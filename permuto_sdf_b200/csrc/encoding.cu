// Multi-resolution permutohedral-lattice hash encoding for sm_90a: forward (barycentric gather),
// backward to the lattice (warp-aggregated vector atomics), backward to positions, and the double
// backward needed by the eikonal / curvature losses.
//
// The algorithm is the one of the external `permutohedral_encoding` package the reference imports
// (permuto_sdf_py/models/models.py:20,149,186); its source is not vendored in the reference, the
// semantics implemented here are the published ones restated in SURVEY.md Appendix B:
// elevate (x+shift)*scale to the hyperplane, round to the remainder-0 lattice point, rank-sort the
// residuals, barycentric weights by rank, hash the D-int key of each of the D+1 simplex vertices
// (h = (h + key_i) * 2531011 over i, mod capacity), blend F features, multiply by the level window.
//
// Every kernel is a template on the input width D in {2..6} and the features per level F in {1, 2, 4, 8}; the
// library instantiates all 20 pairs (with_dim_feat below is the one list of them).
//
// Mapping. One thread per sample, all levels in that thread; a warp is 32 consecutive samples,
// i.e. neighbours on a ray, so on coarse levels the 32 lanes hit the same few F*4-byte table rows (L1
// broadcast) and on fine levels each lane has (D+1)*UNROLL independent gathers in flight against the
// L2-resident table (L*T*F*4 B = 33.5 MB at L=16, F=2 < 50 MB L2). A row is one ld.global.nc of f32, v2 or v4
// (two v4 at F=8). Outputs are staged in shared memory and written as one contiguous [32, C] block per warp.
// The backward reduces duplicates inside the warp (match_any + segmented shuffle tree over the F lanes of
// values) before issuing one red.global.add.{f32,v2.f32,v4.f32} (two v4 at F=8) per distinct vertex.
// Position gradients need no atomics because a thread owns all levels of its sample.
//
// Deterministic variants (k_fx_enc_backward, k_fx_enc_double_backward): the same kernels with the lattice scatter in 64-bit fixed
// point. Each contribution is rounded to the 2^-34 grid (fx_of) before anything is added to it; the peers' integers are summed with
// 64-bit shuffles and one red.global.add.u64 per feature and distinct vertex adds them to caller-owned accumulators, which k_fx_flush
// adds to the float table and clears. Integer addition is associative, so the lattice gradient depends only on the multiset of
// (position, upstream gradient) rows, not on their order, the warp layout or the run. The float kernels are left as they are: these are
// separate kernels rather than a template parameter of them, so the float kernels keep their names and their SASS.
#include "common.cuh"
#include "../../include/psdf_b200.h"

#include <type_traits>
#include <utility>

using namespace psdf;

namespace {
constexpr unsigned kFull = 0xffffffffu;
constexpr int kEncThreads = 128;
constexpr int kGroups = kEncThreads / 32;   // level groups (warps) per block; a block covers 32 samples
constexpr int kMaxLevels = 32;

struct EncParams {
    int N, L, T, C;          // samples, levels, table capacity, output columns
    int concat;              // concat raw points
    float points_scaling;
    unsigned cap_mask;       // floor(2^32 / T): multiplier of the division-free h mod T (see vertex_index)
};

// Levels in flight per thread (unroll of the level loop): 4 in the forward, 2 in both backward kernels, as at F = 2, except where ptxas
// spills at that unroll (CUDA 12.9, sm_90a; chosen from its -v report, checked by tests/test_encoding_dims_cpu.py): the forward at
// (4, 8) and (5, 8), the backward at (6, 2), the double backward at F = 8.
template <int D, int F> constexpr int kFwdUnroll = (F == 8 && (D == 4 || D == 5)) ? 2 : 4;
template <int D, int F> constexpr int kBwdUnroll = (D == 6 && F == 2) ? 1 : 2;
template <int D, int F> constexpr int kDblUnroll = F == 8 ? 1 : 2;
// The fixed-point variants hold F 64-bit partial sums per vertex in the peer reduction; lowered from 2 to 1 where ptxas spills at 2: the
// backward at (3, 1), (3, 2), (4, 2) and (6, 2), the double backward at F >= 4 and at (5, 2).
template <int D, int F> constexpr int kFxBwdUnroll = ((D == 3 && F <= 2) || (D == 4 && F == 2) || (D == 6 && F == 2)) ? 1 : 2;
template <int D, int F> constexpr int kFxDblUnroll = (F >= 4 || (D == 5 && F == 2)) ? 1 : 2;

template <int D>
struct Simplex {
    int rem0[D + 1];
    int rank[D + 1];
    float bary[D + 2];
};

// elevation of a D-vector of (already scaled) coordinates to the (D+1)-dim hyperplane
template <int D>
__device__ __forceinline__ void elevate(const float* cf, float* elevated) {
    float sm = 0.0f;
#pragma unroll
    for (int i = D; i > 0; i--) {
        elevated[i] = __fmaf_rn(-(float)i, cf[i - 1], sm);
        sm = __fadd_rn(sm, cf[i - 1]);
    }
    elevated[0] = sm;
}

// locate the enclosing simplex: remainder-0 point, rank permutation and barycentric weights
template <int D>
__device__ __forceinline__ void locate(const float* elevated, Simplex<D>& s) {
    const float inv = 1.0f / (float)(D + 1);
    int sum = 0;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float v = __fmul_rn(elevated[i], inv);
        float up = __fmul_rn(ceilf(v), (float)(D + 1));
        float down = __fmul_rn(floorf(v), (float)(D + 1));
        s.rem0[i] = (__fsub_rn(up, elevated[i]) < __fsub_rn(elevated[i], down)) ? (int)up : (int)down;
        sum += s.rem0[i];
        s.rank[i] = 0;
    }
    sum /= (D + 1);
#pragma unroll
    for (int i = 0; i < D; i++) {
        float di = __fsub_rn(elevated[i], (float)s.rem0[i]);
#pragma unroll
        for (int j = i + 1; j <= D; j++) {
            if (di < __fsub_rn(elevated[j], (float)s.rem0[j])) s.rank[i]++; else s.rank[j]++;
        }
    }
#pragma unroll
    for (int i = 0; i <= D; i++) {
        s.rank[i] += sum;
        if (s.rank[i] < 0) { s.rank[i] += D + 1; s.rem0[i] += D + 1; }
        else if (s.rank[i] > D) { s.rank[i] -= D + 1; s.rem0[i] -= D + 1; }
    }
#pragma unroll
    for (int i = 0; i <= D + 1; i++) s.bary[i] = 0.0f;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float delta = __fmul_rn(__fsub_rn(elevated[i], (float)s.rem0[i]), inv);
        // bary[D - rank] += delta ; bary[D + 1 - rank] -= delta   (static indexing to stay in registers)
#pragma unroll
        for (int r = 0; r <= D + 1; r++) {
            if (r == D - s.rank[i]) s.bary[r] = __fadd_rn(s.bary[r], delta);
            if (r == D + 1 - s.rank[i]) s.bary[r] = __fsub_rn(s.bary[r], delta);
        }
    }
    s.bary[0] = __fadd_rn(s.bary[0], __fadd_rn(1.0f, s.bary[D + 1]));
}

// d(bary)/d(direction): same scatter as the weights, applied to the elevated direction (weights are
// piecewise linear in x, so this is exact inside a simplex)
template <int D>
__device__ __forceinline__ void bary_tangent(const float* d_elev, const Simplex<D>& s, float* db) {
    const float inv = 1.0f / (float)(D + 1);
#pragma unroll
    for (int i = 0; i <= D + 1; i++) db[i] = 0.0f;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float delta = d_elev[i] * inv;
#pragma unroll
        for (int r = 0; r <= D + 1; r++) {
            if (r == D - s.rank[i]) db[r] += delta;
            if (r == D + 1 - s.rank[i]) db[r] -= delta;
        }
    }
    db[0] += db[D + 1];
}

template <int D>
__device__ __forceinline__ unsigned vertex_index(const Simplex<D>& s, int r, const EncParams& p) {
    unsigned h = 0;
#pragma unroll
    for (int i = 0; i < D; i++) {
        int key = s.rem0[i] + r;
        if (s.rank[i] > D - r) key -= (D + 1);
        h += (unsigned)key;
        h *= 2531011u;
    }
    // h mod T without a division: umulhi(h, floor(2^32 / T)) is the quotient or one less -> one conditional subtraction
    const unsigned rem = h - __umulhi(h, p.cap_mask) * (unsigned)p.T;
    return rem >= (unsigned)p.T ? rem - (unsigned)p.T : rem;
}

// reverse of locate()'s weight scatter + elevation: dL/dbary[0..D] -> dL/dx (before the per-dim scale)
template <int D>
__device__ __forceinline__ void bary_grad_to_cf(float* dB /* size D+2, dB[D+1] must be 0 on entry */, const Simplex<D>& s,
                                                float* dcf) {
    const float inv = 1.0f / (float)(D + 1);
    dB[D + 1] += dB[0];
    float de[D + 1];
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float a = 0.0f, b = 0.0f;
#pragma unroll
        for (int r = 0; r <= D + 1; r++) {
            if (r == D - s.rank[i]) a = dB[r];
            if (r == D + 1 - s.rank[i]) b = dB[r];
        }
        de[i] = (a - b) * inv;
    }
    // elevated[0] = sum_k cf[k]; elevated[i] = sum_{k>=i} cf[k] - i*cf[i-1]
    float run = 0.0f;
#pragma unroll
    for (int k = 0; k < D; k++) {
        run += de[k];
        dcf[k] = run - (float)(k + 1) * de[k + 1];
    }
}

// one table row of F floats: its vector type, and one ld.global.nc per 16 bytes (F = 8: two v4)
struct float8 { float4 lo, hi; };
template <int F> struct RowOf;
template <> struct RowOf<1> { using T = float; };
template <> struct RowOf<2> { using T = float2; };
template <> struct RowOf<4> { using T = float4; };
template <> struct RowOf<8> { using T = float8; };
template <int F> using Row = typename RowOf<F>::T;

template <int F>
__device__ __forceinline__ void load_row(const Row<F>* p, float (&v)[F]) {
    if constexpr (F == 1) {
        v[0] = __ldg(p);
    } else if constexpr (F == 2) {
        float2 t = __ldg(p);
        v[0] = t.x; v[1] = t.y;
    } else {
        const float4* q = reinterpret_cast<const float4*>(p);
#pragma unroll
        for (int k = 0; k < F / 4; k++) {
            float4 t = __ldg(q + k);
            v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
        }
    }
}

// F floats held in registers, passed by value like the float2 of the F = 2 kernels
template <int F>
struct Feat {
    float v[F];
};
// op(0), ..., op(F - 1) as straight-line code (no loop for the optimizer to rotate or unroll late)
template <typename Op, int... K>
__device__ __forceinline__ void each_feat(Op&& op, std::integer_sequence<int, K...>) {
    (op(K), ...);
}
template <int F, typename Op>
__device__ __forceinline__ void each_feat(Op&& op) {
    each_feat(op, std::make_integer_sequence<int, F>{});
}

// segmented sum over lanes that share a key (peers mask from __match_any_sync); result valid in the first peer
template <int F>
__device__ __forceinline__ Feat<F> add_peers(unsigned peers, Feat<F> x, int lane) {
    int rel = __popc(peers << (31 - lane) << 1);  // peers below me
    peers &= (0xfffffffeu << lane);
    while (__any_sync(kFull, peers)) {
        int next = __ffs(peers);
        Feat<F> t;
        each_feat<F>([&](int k) { t.v[k] = __shfl_sync(kFull, x.v[k], (next - 1) & 31); });
        if (next) each_feat<F>([&](int k) { x.v[k] += t.v[k]; });
        int done = rel & 1;
        peers &= __ballot_sync(kFull, !done);
        rel >>= 1;
    }
    return x;
}
// F fixed-point values (fx_of) held in registers
template <int F>
struct FeatFx {
    unsigned long long v[F];
};
// add_peers on integers: wrap-around addition is exact and associative, so the sums do not depend on the order of the peers
template <int F>
__device__ __forceinline__ FeatFx<F> add_peers(unsigned peers, FeatFx<F> x, int lane) {
    int rel = __popc(peers << (31 - lane) << 1);
    peers &= (0xfffffffeu << lane);
    while (__any_sync(kFull, peers)) {
        int next = __ffs(peers);
        FeatFx<F> t;
        each_feat<F>([&](int k) { t.v[k] = __shfl_sync(kFull, x.v[k], (next - 1) & 31); });
        if (next) each_feat<F>([&](int k) { x.v[k] += t.v[k]; });
        int done = rel & 1;
        peers &= __ballot_sync(kFull, !done);
        rel >>= 1;
    }
    return x;
}
// the contributions c of this lane's sample (valid) to row idx of one level's accumulators: rounded to fixed point, summed over the
// lanes that share the row, added by the first of them with F scalar reductions (PTX has no vector u64 red)
template <int F>
__device__ __forceinline__ void scatter_row_fx(unsigned long long* acc, unsigned idx, bool valid, const Feat<F>& c, int lane) {
    FeatFx<F> q;
    each_feat<F>([&](int k) { q.v[k] = fx_of(c.v[k]); });
    unsigned key = valid ? idx : 0xffffffffu;
    unsigned peers = __match_any_sync(kFull, key);
    q = add_peers<F>(peers, q, lane);
    if (valid && lane == __ffs(peers) - 1) {
        unsigned long long* row = acc + (size_t)idx * F;
        each_feat<F>([&](int k) { asm volatile("red.global.add.u64 [%0], %1;" ::"l"(row + k), "l"(q.v[k]) : "memory"); });
    }
}
// one vector reduction per 16 bytes of the row (F * 4 bytes, 16-byte aligned for F >= 4)
template <int F>
__device__ __forceinline__ void red_add(float* addr, Feat<F> x) {
    if constexpr (F == 1) {
        asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(x.v[0]) : "memory");
    } else if constexpr (F == 2) {
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(x.v[0]), "f"(x.v[1]) : "memory");
    } else {
#pragma unroll
        for (int k = 0; k < F; k += 4)
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr + k), "f"(x.v[k]), "f"(x.v[k + 1]), "f"(x.v[k + 2]),
                         "f"(x.v[k + 3]) : "memory");
    }
}

// per-level scale / shift with a fixed stride per level: 4 floats up to D = 4, 8 for D = 5, 6
template <int D>
struct LevelConsts {
    static constexpr int S = D <= 4 ? 4 : 8;
    float scale[kMaxLevels * S];
    float shift[kMaxLevels * S];
    float window[kMaxLevels];
};
template <int D>
__device__ __forceinline__ void load_level_consts(LevelConsts<D>& lc, const float* __restrict__ scale,
                                                  const float* __restrict__ shift, const float* __restrict__ window, int L) {
    constexpr int S = LevelConsts<D>::S;
    for (int i = threadIdx.x; i < L * D; i += blockDim.x) {
        lc.scale[(i / D) * S + (i % D)] = scale[i];
        lc.shift[(i / D) * S + (i % D)] = shift ? shift[i] : 0.0f;
    }
    for (int i = threadIdx.x; i < L; i += blockDim.x) lc.window[i] = window ? window[i] : 1.0f;
}

// ------------------------------------------------------------------------------------------------ forward
template <int D, int F>
__global__ void __launch_bounds__(kEncThreads)
k_enc_forward(EncParams p, const float* __restrict__ pos, const Row<F>* __restrict__ lattice, const float* __restrict__ scale,
              const float* __restrict__ shift, const float* __restrict__ window, float* __restrict__ out) {
    // block = 32 consecutive samples x 4 level groups: warp g handles levels g, g+4, ... of the same 32 samples
    constexpr int S = LevelConsts<D>::S;
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts<D> lc;
    load_level_consts<D>(lc, scale, shift, window, p.L);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;                      // +1 float: conflict-free column writes
    float* tile = smem_dyn;
    const int n = blockIdx.x * 32 + lane;
    const bool valid = n < p.N;
    float x[D];
#pragma unroll
    for (int i = 0; i < D; i++) x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;

#pragma unroll kFwdUnroll<D, F>
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], elevated[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * S + i]), lc.scale[l * S + i]);
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        const Row<F>* tab = lattice + (size_t)l * p.T;
        float v[D + 1][F];
#pragma unroll
        for (int r = 0; r <= D; r++) load_row<F>(tab + vertex_index<D>(s, r, p), v[r]);
        float w = lc.window[l];
        float a[F];
#pragma unroll
        for (int k = 0; k < F; k++) a[k] = 0.0f;
#pragma unroll
        for (int r = 0; r <= D; r++) {
            float wr = s.bary[r] * w;
#pragma unroll
            for (int k = 0; k < F; k++) a[k] = fmaf(v[r][k], wr, a[k]);
        }
#pragma unroll
        for (int k = 0; k < F; k++) tile[lane * stride + F * l + k] = a[k];
    }
    if (p.concat && warp == kGroups - 1) {
        const int base = F * p.L;
        for (int c = base; c < p.C; c++) {
            int d = c - base;
            float val = 0.0f;
#pragma unroll
            for (int i = 0; i < D; i++) if (i == d) val = x[i] * p.points_scaling;
            tile[lane * stride + c] = val;
        }
    }
    __syncthreads();
    // contiguous [rows, C] block of this CTA, written by all 128 threads
    const int row0 = blockIdx.x * 32;
    const int rows = min(32, p.N - row0);
    float* dst = out + (size_t)row0 * p.C;
    const int total = rows * p.C;
    for (int e = threadIdx.x; e < total; e += kEncThreads) {
        int r = e / p.C, c = e - r * p.C;
        dst[e] = tile[r * stride + c];
    }
}

// ------------------------------------------------------------------------------------------------ backward
// grad_lattice[l][idx][:] += window_l * bary_r * g[n][l][:]         (warp aggregated vector red)
// grad_pos[n][j]          = sum_l window_l * sum_r (val_r . g_l) dB_r/dx_j  (+ concat columns)
template <int D, int F, bool LATTICE, bool POS>
__global__ void __launch_bounds__(kEncThreads)
k_enc_backward(EncParams p, const float* __restrict__ pos, const Row<F>* __restrict__ lattice, const float* __restrict__ scale,
               const float* __restrict__ shift, const float* __restrict__ window, const float* __restrict__ grad_out,
               float* __restrict__ grad_lattice, float* __restrict__ grad_pos) {
    constexpr int S = LevelConsts<D>::S;
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts<D> lc;
    __shared__ float red[kGroups][32][S];
    load_level_consts<D>(lc, scale, shift, window, p.L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;
    float* gtile = smem_dyn;                         // staged [32, C] block of grad_out (coalesced read)
    const int row0 = blockIdx.x * 32;
    {
        const int rows = min(32, p.N - row0);
        const float* src = grad_out + (size_t)row0 * p.C;
        for (int e = threadIdx.x; e < 32 * p.C; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            gtile[r * stride + c] = (r < rows) ? src[e] : 0.0f;
        }
    }
    __syncthreads();
    const int n = row0 + lane;
    const bool valid = n < p.N;
    float x[D], gp[D];
#pragma unroll
    for (int i = 0; i < D; i++) { x[i] = valid ? pos[(size_t)n * D + i] : 0.0f; gp[i] = 0.0f; }
    const float* g_row = gtile + lane * stride;

#pragma unroll kBwdUnroll<D, F>
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], elevated[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * S + i]), lc.scale[l * S + i]);
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        float g[F];
        each_feat<F>([&](int k) { g[k] = g_row[F * l + k]; });
        float w = lc.window[l];
        unsigned idx[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) idx[r] = vertex_index<D>(s, r, p);
        if (POS) {
            const Row<F>* tab = lattice + (size_t)l * p.T;
            float dB[D + 2];
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float v[F];
                load_row<F>(tab + idx[r], v);
                float dot = v[0] * g[0];
                each_feat<F - 1>([&](int k) { dot = dot + v[k + 1] * g[k + 1]; });
                dB[r] = w * dot;
            }
            dB[D + 1] = 0.0f;
            float dcf[D];
            bary_grad_to_cf<D>(dB, s, dcf);
#pragma unroll
            for (int i = 0; i < D; i++) gp[i] = fmaf(dcf[i], lc.scale[l * S + i], gp[i]);
        }
        if (LATTICE) {
            float* gtab = grad_lattice + (size_t)l * p.T * F;
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float wr = s.bary[r] * w;
                Feat<F> c;
#pragma unroll
                for (int k = 0; k < F; k++) c.v[k] = g[k] * wr;
                unsigned key = valid ? idx[r] : 0xffffffffu;
                unsigned peers = __match_any_sync(kFull, key);
                c = add_peers<F>(peers, c, lane);
                if (valid && lane == __ffs(peers) - 1) red_add<F>(gtab + (size_t)idx[r] * F, c);
            }
        }
    }
    if (POS) {
        // sum the per-level-group partial position gradients of the 4 warps
#pragma unroll
        for (int i = 0; i < D; i++) red[warp][lane][i] = gp[i];
        __syncthreads();
        if (warp == 0 && valid) {
#pragma unroll
            for (int i = 0; i < D; i++) {
                float acc = red[0][lane][i];
#pragma unroll
                for (int w2 = 1; w2 < kGroups; w2++) acc += red[w2][lane][i];
                if (p.concat && F * p.L + i < p.C) acc = fmaf(g_row[F * p.L + i], p.points_scaling, acc);
                grad_pos[(size_t)n * D + i] = acc;
            }
        }
    }
}

// the backward with the lattice gradient in fixed point: k_enc_backward<D, F, true, POS> with the scatter into the accumulators fx
// [L, T, F] (scatter_row_fx); grad_pos is formed by the same operations, so it is the float kernel's bit for bit
template <int D, int F, bool POS>
__global__ void __launch_bounds__(kEncThreads)
k_fx_enc_backward(EncParams p, const float* __restrict__ pos, const Row<F>* __restrict__ lattice, const float* __restrict__ scale,
                  const float* __restrict__ shift, const float* __restrict__ window, const float* __restrict__ grad_out,
                  unsigned long long* __restrict__ fx, float* __restrict__ grad_pos) {
    constexpr int S = LevelConsts<D>::S;
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts<D> lc;
    __shared__ float red[kGroups][32][S];
    load_level_consts<D>(lc, scale, shift, window, p.L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;
    float* gtile = smem_dyn;
    const int row0 = blockIdx.x * 32;
    {
        const int rows = min(32, p.N - row0);
        const float* src = grad_out + (size_t)row0 * p.C;
        for (int e = threadIdx.x; e < 32 * p.C; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            gtile[r * stride + c] = (r < rows) ? src[e] : 0.0f;
        }
    }
    __syncthreads();
    const int n = row0 + lane;
    const bool valid = n < p.N;
    float x[D], gp[D];
#pragma unroll
    for (int i = 0; i < D; i++) { x[i] = valid ? pos[(size_t)n * D + i] : 0.0f; gp[i] = 0.0f; }
    const float* g_row = gtile + lane * stride;

#pragma unroll kFxBwdUnroll<D, F>
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], elevated[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * S + i]), lc.scale[l * S + i]);
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        float g[F];
        each_feat<F>([&](int k) { g[k] = g_row[F * l + k]; });
        float w = lc.window[l];
        unsigned idx[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) idx[r] = vertex_index<D>(s, r, p);
        if (POS) {
            const Row<F>* tab = lattice + (size_t)l * p.T;
            float dB[D + 2];
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float v[F];
                load_row<F>(tab + idx[r], v);
                float dot = v[0] * g[0];
                each_feat<F - 1>([&](int k) { dot = dot + v[k + 1] * g[k + 1]; });
                dB[r] = w * dot;
            }
            dB[D + 1] = 0.0f;
            float dcf[D];
            bary_grad_to_cf<D>(dB, s, dcf);
#pragma unroll
            for (int i = 0; i < D; i++) gp[i] = fmaf(dcf[i], lc.scale[l * S + i], gp[i]);
        }
        unsigned long long* acc = fx + (size_t)l * p.T * F;
#pragma unroll
        for (int r = 0; r <= D; r++) {
            float wr = s.bary[r] * w;
            Feat<F> c;
#pragma unroll
            for (int k = 0; k < F; k++) c.v[k] = g[k] * wr;
            scatter_row_fx<F>(acc, idx[r], valid, c, lane);
        }
    }
    if (POS) {
#pragma unroll
        for (int i = 0; i < D; i++) red[warp][lane][i] = gp[i];
        __syncthreads();
        if (warp == 0 && valid) {
#pragma unroll
            for (int i = 0; i < D; i++) {
                float acc = red[0][lane][i];
#pragma unroll
                for (int w2 = 1; w2 < kGroups; w2++) acc += red[w2][lane][i];
                if (p.concat && F * p.L + i < p.C) acc = fmaf(g_row[F * p.L + i], p.points_scaling, acc);
                grad_pos[(size_t)n * D + i] = acc;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ double backward
// Upstream gradient gg[n][j] flows into grad_pos. With dB_r = sum_j gg_j dB_r/dx_j (tangent of the weights):
//   grad_lattice[l][idx_r][:] += window_l * dB_r * g[n][l][:]
//   grad_grad_out[n][l][:]     = window_l * sum_r dB_r * val_r[:]      (concat columns: gg_j * scaling)
template <int D, int F, bool LATTICE, bool GOUT>
__global__ void __launch_bounds__(kEncThreads)
k_enc_double_backward(EncParams p, const float* __restrict__ pos, const Row<F>* __restrict__ lattice,
                      const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ window,
                      const float* __restrict__ gg_pos, const float* __restrict__ grad_out, float* __restrict__ grad_lattice,
                      float* __restrict__ grad_grad_out) {
    constexpr int S = LevelConsts<D>::S;
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts<D> lc;
    load_level_consts<D>(lc, scale, shift, window, p.L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;
    float* gtile = smem_dyn;                         // staged grad_out block
    float* otile = smem_dyn + 32 * stride;           // grad_grad_out block, written out coalesced
    const int row0 = blockIdx.x * 32;
    const int rows = min(32, p.N - row0);
    if (LATTICE) {
        const float* src = grad_out + (size_t)row0 * p.C;
        for (int e = threadIdx.x; e < 32 * p.C; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            gtile[r * stride + c] = (r < rows) ? src[e] : 0.0f;
        }
    }
    __syncthreads();
    const int n = row0 + lane;
    const bool valid = n < p.N;
    float x[D], u[D];
#pragma unroll
    for (int i = 0; i < D; i++) {
        x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;
        u[i] = valid ? gg_pos[(size_t)n * D + i] : 0.0f;
    }
#pragma unroll kDblUnroll<D, F>
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], dcf[D], elevated[D + 1], d_elev[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) {
            cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * S + i]), lc.scale[l * S + i]);
            dcf[i] = u[i] * lc.scale[l * S + i];
        }
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        {
            float sm = 0.0f;
#pragma unroll
            for (int i = D; i > 0; i--) { d_elev[i] = sm - (float)i * dcf[i - 1]; sm += dcf[i - 1]; }
            d_elev[0] = sm;
        }
        float db[D + 2];
        bary_tangent<D>(d_elev, s, db);
        float w = lc.window[l];
        unsigned idx[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) idx[r] = vertex_index<D>(s, r, p);
        if (GOUT) {
            const Row<F>* tab = lattice + (size_t)l * p.T;
            float a[F];
            each_feat<F>([&](int k) { a[k] = 0.0f; });
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float v[F];
                load_row<F>(tab + idx[r], v);
                float c = db[r] * w;
                each_feat<F>([&](int k) { a[k] = fmaf(v[k], c, a[k]); });
            }
            each_feat<F>([&](int k) { otile[lane * stride + F * l + k] = a[k]; });
        }
        if (LATTICE) {
            float g[F];
            each_feat<F>([&](int k) { g[k] = gtile[lane * stride + F * l + k]; });
            float* gtab = grad_lattice + (size_t)l * p.T * F;
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float c = db[r] * w;
                Feat<F> cv;
#pragma unroll
                for (int k = 0; k < F; k++) cv.v[k] = g[k] * c;
                unsigned key = valid ? idx[r] : 0xffffffffu;
                unsigned peers = __match_any_sync(kFull, key);
                cv = add_peers<F>(peers, cv, lane);
                if (valid && lane == __ffs(peers) - 1) red_add<F>(gtab + (size_t)idx[r] * F, cv);
            }
        }
    }
    if (GOUT) {
        if (p.concat && warp == kGroups - 1) {
            const int base = F * p.L;
            for (int c = base; c < p.C; c++) {
                int d = c - base;
                float val = 0.0f;
#pragma unroll
                for (int i = 0; i < D; i++) if (i == d) val = u[i] * p.points_scaling;
                otile[lane * stride + c] = val;
            }
        }
        __syncthreads();
        float* dst = grad_grad_out + (size_t)row0 * p.C;
        const int total = rows * p.C;
        for (int e = threadIdx.x; e < total; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            dst[e] = otile[r * stride + c];
        }
    }
}

// the double backward with the lattice term in fixed point: k_enc_double_backward<D, F, true, GOUT> with the scatter into the
// accumulators fx [L, T, F]; grad_grad_out is formed by the same operations, so it is the float kernel's bit for bit
template <int D, int F, bool GOUT>
__global__ void __launch_bounds__(kEncThreads)
k_fx_enc_double_backward(EncParams p, const float* __restrict__ pos, const Row<F>* __restrict__ lattice,
                         const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ window,
                         const float* __restrict__ gg_pos, const float* __restrict__ grad_out, unsigned long long* __restrict__ fx,
                         float* __restrict__ grad_grad_out) {
    constexpr int S = LevelConsts<D>::S;
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts<D> lc;
    load_level_consts<D>(lc, scale, shift, window, p.L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;
    float* gtile = smem_dyn;
    float* otile = smem_dyn + 32 * stride;
    const int row0 = blockIdx.x * 32;
    const int rows = min(32, p.N - row0);
    {
        const float* src = grad_out + (size_t)row0 * p.C;
        for (int e = threadIdx.x; e < 32 * p.C; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            gtile[r * stride + c] = (r < rows) ? src[e] : 0.0f;
        }
    }
    __syncthreads();
    const int n = row0 + lane;
    const bool valid = n < p.N;
    float x[D], u[D];
#pragma unroll
    for (int i = 0; i < D; i++) {
        x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;
        u[i] = valid ? gg_pos[(size_t)n * D + i] : 0.0f;
    }
#pragma unroll kFxDblUnroll<D, F>
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], dcf[D], elevated[D + 1], d_elev[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) {
            cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * S + i]), lc.scale[l * S + i]);
            dcf[i] = u[i] * lc.scale[l * S + i];
        }
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        {
            float sm = 0.0f;
#pragma unroll
            for (int i = D; i > 0; i--) { d_elev[i] = sm - (float)i * dcf[i - 1]; sm += dcf[i - 1]; }
            d_elev[0] = sm;
        }
        float db[D + 2];
        bary_tangent<D>(d_elev, s, db);
        float w = lc.window[l];
        unsigned idx[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) idx[r] = vertex_index<D>(s, r, p);
        if (GOUT) {
            const Row<F>* tab = lattice + (size_t)l * p.T;
            float a[F];
            each_feat<F>([&](int k) { a[k] = 0.0f; });
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float v[F];
                load_row<F>(tab + idx[r], v);
                float c = db[r] * w;
                each_feat<F>([&](int k) { a[k] = fmaf(v[k], c, a[k]); });
            }
            each_feat<F>([&](int k) { otile[lane * stride + F * l + k] = a[k]; });
        }
        float g[F];
        each_feat<F>([&](int k) { g[k] = gtile[lane * stride + F * l + k]; });
        unsigned long long* acc = fx + (size_t)l * p.T * F;
#pragma unroll
        for (int r = 0; r <= D; r++) {
            float c = db[r] * w;
            Feat<F> cv;
#pragma unroll
            for (int k = 0; k < F; k++) cv.v[k] = g[k] * c;
            scatter_row_fx<F>(acc, idx[r], valid, cv, lane);
        }
    }
    if (GOUT) {
        if (p.concat && warp == kGroups - 1) {
            const int base = F * p.L;
            for (int c = base; c < p.C; c++) {
                int d = c - base;
                float val = 0.0f;
#pragma unroll
                for (int i = 0; i < D; i++) if (i == d) val = u[i] * p.points_scaling;
                otile[lane * stride + c] = val;
            }
        }
        __syncthreads();
        float* dst = grad_grad_out + (size_t)row0 * p.C;
        const int total = rows * p.C;
        for (int e = threadIdx.x; e < total; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            dst[e] = otile[r * stride + c];
        }
    }
}

// The (D, F) pairs the library is built for: fn(integral_constant D, integral_constant F) runs for one of them and the call returns
// true; any other pair returns false without calling fn. This switch is the only list of the supported pairs.
template <int D, typename Fn>
inline bool with_feat(int F, Fn&& fn) {
    using std::integral_constant;
    switch (F) {
        case 1: fn(integral_constant<int, D>{}, integral_constant<int, 1>{}); return true;
        case 2: fn(integral_constant<int, D>{}, integral_constant<int, 2>{}); return true;
        case 4: fn(integral_constant<int, D>{}, integral_constant<int, 4>{}); return true;
        case 8: fn(integral_constant<int, D>{}, integral_constant<int, 8>{}); return true;
        default: return false;
    }
}
template <typename Fn>
inline bool with_dim_feat(int D, int F, Fn&& fn) {
    switch (D) {
        case 2: return with_feat<2>(F, fn);
        case 3: return with_feat<3>(F, fn);
        case 4: return with_feat<4>(F, fn);
        case 5: return with_feat<5>(F, fn);
        case 6: return with_feat<6>(F, fn);
        default: return false;
    }
}

inline int make_params(EncParams& p, int N, int D, int L, int F, int T, int concat, float points_scaling) {
    if (!with_dim_feat(D, F, [](auto, auto) {}) || L < 1 || L > kMaxLevels || T < 1) return PSDF_ERR_UNSUPPORTED;
    p.N = N; p.L = L; p.T = T;
    int E = concat ? (D + F - 1) / F : 0;
    p.C = (L + E) * F;
    p.concat = concat;
    p.points_scaling = points_scaling;
    p.cap_mask = T <= 1 ? 0xffffffffu : (unsigned)(0x100000000ull / (unsigned long long)(unsigned)T);
    return PSDF_OK;
}
// table rows are read and reduced as F * 4-byte vectors (16-byte pieces for F >= 4)
inline bool rows_aligned(const void* a, int F) { return ((uintptr_t)a % (size_t)(F < 4 ? F * 4 : 16)) == 0; }

// Dynamic shared memory is 32 * (C + 1) floats per staged tile, C = (L + E) * F; at F = 8 and L = 32 the double backward's two tiles
// take 66 KB. A kernel asked for more than this opts in (once per device) to as much as the device allows beside its static shared
// memory; smaller launches (every F <= 4 call) leave the kernel's attributes as they are.
constexpr size_t kSmemOptInAbove = 32 * 1024;
template <auto Kernel, typename... Args>
inline void launch(int blocks, size_t smem, cudaStream_t stream, Args... args) {
    static bool slot[64];
    if (smem > kSmemOptInAbove) psdf_optin_smem(Kernel, 227 * 1024, slot);
    Kernel<<<blocks, kEncThreads, smem, stream>>>(args...);
}
#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {

int psdf_enc_forward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                     const float* shift, const float* window, int concat_points, float points_scaling, float* out, void* stream) {
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (N == 0) return PSDF_OK;
    if (!rows_aligned(lattice, F)) return PSDF_ERR_ARG;
    int blocks = div_up(N, 32);
    size_t smem = (size_t)32 * (p.C + 1) * sizeof(float);
    with_dim_feat(D, F, [&](auto d, auto f) {
        constexpr int DD = decltype(d)::value, FF = decltype(f)::value;
        launch<k_enc_forward<DD, FF>>(blocks, smem, ST, p, pos, reinterpret_cast<const Row<FF>*>(lattice), scale_factor, shift, window, out);
    });
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_enc_backward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                      const float* shift, const float* window, int concat_points, float points_scaling, const float* grad_out,
                      float* grad_lattice, float* grad_pos, void* stream) {
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (N == 0 || (!grad_lattice && !grad_pos)) return PSDF_OK;
    if (!rows_aligned(lattice, F) || !rows_aligned(grad_lattice, F)) return PSDF_ERR_ARG;
    int blocks = div_up(N, 32);
    size_t smem = (size_t)32 * (p.C + 1) * sizeof(float);
    with_dim_feat(D, F, [&](auto d, auto f) {
        constexpr int DD = decltype(d)::value, FF = decltype(f)::value;
        const Row<FF>* lat = reinterpret_cast<const Row<FF>*>(lattice);
#define LAUNCH_BWD(LA, PO) \
    launch<k_enc_backward<DD, FF, LA, PO>>(blocks, smem, ST, p, pos, lat, scale_factor, shift, window, grad_out, grad_lattice, grad_pos)
        if (grad_lattice && grad_pos) LAUNCH_BWD(true, true);
        else if (grad_lattice) LAUNCH_BWD(true, false);
        else LAUNCH_BWD(false, true);
#undef LAUNCH_BWD
    });
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_enc_double_backward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                             const float* shift, const float* window, int concat_points, float points_scaling,
                             const float* gg_pos, const float* grad_out, float* grad_lattice, float* grad_grad_out, void* stream) {
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (N == 0 || (!grad_lattice && !grad_grad_out)) return PSDF_OK;
    if (!rows_aligned(lattice, F) || !rows_aligned(grad_lattice, F)) return PSDF_ERR_ARG;
    int blocks = div_up(N, 32);
    size_t smem = (size_t)2 * 32 * (p.C + 1) * sizeof(float);
    with_dim_feat(D, F, [&](auto d, auto f) {
        constexpr int DD = decltype(d)::value, FF = decltype(f)::value;
        const Row<FF>* lat = reinterpret_cast<const Row<FF>*>(lattice);
#define LAUNCH_DBL(LA, GO)                                                                                                         \
    launch<k_enc_double_backward<DD, FF, LA, GO>>(blocks, smem, ST, p, pos, lat, scale_factor, shift, window, gg_pos, grad_out, grad_lattice, \
                                                  grad_grad_out)
        if (grad_lattice && grad_grad_out) LAUNCH_DBL(true, true);
        else if (grad_lattice) LAUNCH_DBL(true, false);
        else LAUNCH_DBL(false, true);
#undef LAUNCH_DBL
    });
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// The deterministic twins: the lattice gradient is summed in the caller's zeroed fixed-point accumulators fx_lattice [L, T, F], then
// k_fx_flush adds the totals to grad_lattice and clears the accumulators again. Without grad_lattice they are the float entry points.
static int fx_flush_lattice(unsigned long long* fx, float* grad_lattice, const EncParams& p, int F, cudaStream_t stream) {
    FxSegs S;
    S.add(fx, grad_lattice, (long long)p.L * p.T * F);
    return fx_flush(S, stream) ? PSDF_ERR_LAUNCH : PSDF_OK;
}

int psdf_enc_backward_fx(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                         const float* shift, const float* window, int concat_points, float points_scaling, const float* grad_out,
                         float* grad_lattice, float* grad_pos, uint64_t* fx_lattice, void* stream) {
    if (!grad_lattice)
        return psdf_enc_backward(N, D, L, F, T, pos, lattice, scale_factor, shift, window, concat_points, points_scaling, grad_out,
                                 nullptr, grad_pos, stream);
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (!fx_lattice || (uintptr_t)fx_lattice % 8) return PSDF_ERR_ARG;
    if (N == 0) return PSDF_OK;
    if (!rows_aligned(lattice, F) || !rows_aligned(grad_lattice, F)) return PSDF_ERR_ARG;
    unsigned long long* fx = reinterpret_cast<unsigned long long*>(fx_lattice);
    int blocks = div_up(N, 32);
    size_t smem = (size_t)32 * (p.C + 1) * sizeof(float);
    with_dim_feat(D, F, [&](auto d, auto f) {
        constexpr int DD = decltype(d)::value, FF = decltype(f)::value;
        const Row<FF>* lat = reinterpret_cast<const Row<FF>*>(lattice);
#define LAUNCH_FX_BWD(PO) \
    launch<k_fx_enc_backward<DD, FF, PO>>(blocks, smem, ST, p, pos, lat, scale_factor, shift, window, grad_out, fx, grad_pos)
        if (grad_pos) LAUNCH_FX_BWD(true);
        else LAUNCH_FX_BWD(false);
#undef LAUNCH_FX_BWD
    });
    PSDF_CHECK_LAUNCH();
    return fx_flush_lattice(fx, grad_lattice, p, F, ST);
}

int psdf_enc_double_backward_fx(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                                const float* shift, const float* window, int concat_points, float points_scaling,
                                const float* gg_pos, const float* grad_out, float* grad_lattice, float* grad_grad_out,
                                uint64_t* fx_lattice, void* stream) {
    if (!grad_lattice)
        return psdf_enc_double_backward(N, D, L, F, T, pos, lattice, scale_factor, shift, window, concat_points, points_scaling, gg_pos,
                                        grad_out, nullptr, grad_grad_out, stream);
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (!fx_lattice || (uintptr_t)fx_lattice % 8) return PSDF_ERR_ARG;
    if (N == 0) return PSDF_OK;
    if (!rows_aligned(lattice, F) || !rows_aligned(grad_lattice, F)) return PSDF_ERR_ARG;
    unsigned long long* fx = reinterpret_cast<unsigned long long*>(fx_lattice);
    int blocks = div_up(N, 32);
    size_t smem = (size_t)2 * 32 * (p.C + 1) * sizeof(float);
    with_dim_feat(D, F, [&](auto d, auto f) {
        constexpr int DD = decltype(d)::value, FF = decltype(f)::value;
        const Row<FF>* lat = reinterpret_cast<const Row<FF>*>(lattice);
#define LAUNCH_FX_DBL(GO) \
    launch<k_fx_enc_double_backward<DD, FF, GO>>(blocks, smem, ST, p, pos, lat, scale_factor, shift, window, gg_pos, grad_out, fx, grad_grad_out)
        if (grad_grad_out) LAUNCH_FX_DBL(true);
        else LAUNCH_FX_DBL(false);
#undef LAUNCH_FX_DBL
    });
    PSDF_CHECK_LAUNCH();
    return fx_flush_lattice(fx, grad_lattice, p, F, ST);
}

int psdf_abi_version(void) { return PSDF_ABI_VERSION; }
int psdf_device_ok(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); return 0; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, 0) != cudaSuccess) return 0;
    return prop.major == 9 ? 1 : 0;
}

}  // extern "C"
