// Shared pieces of the fused encoding + MLP kernels (fused_sdf.cu: forward / inference, fused_sdf_bwd.cu: training
// backward, fused_rgb*.cu: colour network): MLP operand-blob geometry, permutohedral simplex helpers for D = 3 and 4, the encoder of
// one level and its lattice scatter, GELU and its derivatives, operand tile stores (bf16 hi/lo split in the core-matrix operand
// layout) and the split-product GEMM issue.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "umma.cuh"

namespace psdf_fused {
using namespace psdf;
constexpr int kTile = 128;
constexpr int kMaxLevels = 32;
constexpr int kNL = 4;                 // linear layers of the SDF MLP
constexpr int kATileBytes = 128 * 64 * 2;   // one bf16 operand tile [128 x 64]
constexpr int kLBO = 128;
constexpr int kSBO_A = 1024;           // 8 core matrices (K = 64) per 8-row group
// Accumulator areas (umma.cuh) are sized for one persistent CTA per SM of an H100 SXM (132 SMs), or two for the kernels that run
// two per SM; launches clamp their persistent grids to these counts.
constexpr int kAccCtas = 132;

template <int NL>
struct MlpGeomN {
    int K[NL], N[NL];          // true dims
    int Kp[NL], Np[NL];        // padded dims (K % 16 == 0, N % 16 == 0)
    int w_hi[NL], w_lo[NL], bias[NL];      // byte offsets in the forward blob [0, total)
    int total;
    int t_hi[NL], t_lo[NL];    // byte offsets of the transposed weights W_l^T ([Kp rows][Np cols]) in [total, total + total_t)
    int total_t;
};
using MlpGeom = MlpGeomN<kNL>;
__host__ __device__ inline int pad16(int v) { return (v + 15) & ~15; }
// layer l maps K[l] inputs to N[l] outputs (a plain chain has K[l + 1] == N[l])
template <int NL>
inline MlpGeomN<NL> make_geom_kn(const int* K, const int* N) {
    MlpGeomN<NL> g;
    int off = 0;
    for (int l = 0; l < NL; l++) {
        g.K[l] = K[l]; g.N[l] = N[l];
        g.Kp[l] = pad16(K[l]); g.Np[l] = pad16(N[l]);
        int wbytes = g.Np[l] * g.Kp[l] * 2;
        g.w_hi[l] = off; off += wbytes;
        g.w_lo[l] = off; off += wbytes;
        g.bias[l] = off; off += g.Np[l] * 4;
    }
    g.total = (off + 127) & ~127;
    off = 0;
    for (int l = 0; l < NL; l++) {
        int wbytes = g.Np[l] * g.Kp[l] * 2;
        g.t_hi[l] = off; off += wbytes;
        g.t_lo[l] = off; off += wbytes;
    }
    g.total_t = (off + 127) & ~127;
    return g;
}
inline MlpGeom make_geom_dims(const int* dims) { return make_geom_kn<kNL>(dims, dims + 1); }
inline MlpGeom make_geom(int in_dim, int hidden, int out_dim) {
    int dims[kNL + 1] = {in_dim, hidden, hidden, hidden, out_dim};
    return make_geom_dims(dims);
}

// Element e of layer l: weights [N][K] fp32 (torch.nn.Linear layout) -> hi/lo bf16 in the K-major core-matrix operand layout + fp32 bias;
// second half of the blob: the same weights transposed (rows = input features, K = output features) for the backward GEMMs
// dA = dZ * W. Packed row n holds source row (n + rot) % N (rot = 0: the same order).
template <int NL>
__device__ __forceinline__ void pack_layer_elem(const MlpGeomN<NL>& g, int l, int e, const float* Wl, const float* Bl, uint8_t* blob,
                                                int rot = 0) {
    int total = g.Np[l] * g.Kp[l];
    if (e < total) {
        int n = e / g.Kp[l], k = e - n * g.Kp[l];
        const int src = rot ? (n + rot) % g.N[l] : n;
        float v = (n < g.N[l] && k < g.K[l]) ? Wl[src * g.K[l] + k] : 0.0f;
        __nv_bfloat16 hi, lo;
        umma::split_bf16(v, hi, lo);
        int sbo = (g.Kp[l] / 8) * kLBO;
        int off = (n / 8) * sbo + (k / 8) * kLBO + (n % 8) * 16 + (k % 8) * 2;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.w_hi[l] + off) = hi;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.w_lo[l] + off) = lo;
        // transposed copy: row = k (input feature), reduction index = n (output feature)
        int sbo_t = (g.Np[l] / 8) * kLBO;
        int off_t = (k / 8) * sbo_t + (n / 8) * kLBO + (k % 8) * 16 + (n % 8) * 2;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.total + g.t_hi[l] + off_t) = hi;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.total + g.t_lo[l] + off_t) = lo;
    }
    if (e < g.Np[l]) reinterpret_cast<float*>(blob + g.bias[l])[e] = (e < g.N[l]) ? Bl[rot ? (e + rot) % g.N[l] : e] : 0.0f;
}
static __global__ void k_pack_mlp(MlpGeom g, const float* W0, const float* b0, const float* W1, const float* b1, const float* W2,
                                  const float* b2, const float* W3, const float* b3, uint8_t* blob, int* step_inc = nullptr,
                                  float* it_inc = nullptr) {
    // end-of-iteration bookkeeping folded into the re-pack that closes an optimizer step: AdamW step count and iteration number, both
    // device resident under CUDA-graph replay (every kernel that read them in this iteration has completed: same stream)
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        if (step_inc) step_inc[0] += 1;
        if (it_inc) it_inc[0] += 1.0f;
    }
    const float* W[kNL] = {W0, W1, W2, W3};
    const float* B[kNL] = {b0, b1, b2, b3};
    int l = blockIdx.y;
    pack_layer_elem(g, l, blockIdx.x * blockDim.x + threadIdx.x, W[l], B[l], blob);
}

// ---------------------------------------------------------------------------------------------- lattice helpers (D = 3, 4)
// D = 3: the SDF and colour encoders; D = 4: the background encoder (NeRF++ parametrisation)
template <int D>
struct Simplex { int rem0[D + 1]; int rank[D + 1]; float bary[D + 2]; };
using Simplex3 = Simplex<3>;
template <int D>
__device__ __forceinline__ void elevate(const float* cf, float* e) {
    float sm = 0.0f;
#pragma unroll
    for (int i = D; i > 0; i--) { e[i] = __fmaf_rn(-(float)i, cf[i - 1], sm); sm = __fadd_rn(sm, cf[i - 1]); }
    e[0] = sm;
}
// R[k] = d[i] of the coordinate i whose rank is k (ranks are a permutation of 0..D)
template <int D, int I = 0>
__device__ __forceinline__ float rank_pick(const Simplex<D>& s, const float* d, int k) {
    if constexpr (I == D) return d[D];
    else return s.rank[I] == k ? d[I] : rank_pick<D, I + 1>(s, d, k);
}
template <int D>
__device__ __forceinline__ void by_rank(const Simplex<D>& s, const float* d, float* R) {
#pragma unroll
    for (int k = 0; k <= D; k++) R[k] = rank_pick<D>(s, d, k);
}
template <int D>
__device__ __forceinline__ void locate(const float* e, Simplex<D>& s) {
    constexpr float kInv = 1.0f / (float)(D + 1), kD1 = (float)(D + 1);
    int sum = 0;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float v = __fmul_rn(e[i], kInv);
        // ceil(v) (D+1) == floor(v) (D+1) + D+1 unless v is an integer, where both candidates coincide with e[i] and `down` wins either way
        const float down = __fmul_rn(floorf(v), kD1), up = __fadd_rn(down, kD1);
        s.rem0[i] = (__fsub_rn(up, e[i]) < __fsub_rn(e[i], down)) ? (int)up : (int)down;
        sum += s.rem0[i];
        s.rank[i] = 0;
    }
    sum /= D + 1;
#pragma unroll
    for (int i = 0; i < D; i++) {
        float di = __fsub_rn(e[i], (float)s.rem0[i]);
#pragma unroll
        for (int j = i + 1; j <= D; j++) { if (di < __fsub_rn(e[j], (float)s.rem0[j])) s.rank[i]++; else s.rank[j]++; }
    }
#pragma unroll
    for (int i = 0; i <= D; i++) {
        s.rank[i] += sum;
        if (s.rank[i] < 0) { s.rank[i] += D + 1; s.rem0[i] += D + 1; }
        else if (s.rank[i] > D) { s.rank[i] -= D + 1; s.rem0[i] -= D + 1; }
    }
    // barycentric weights: with R_k the fractional offset of the coordinate of rank k, the reference's scatter
    // (+delta at D - rank, -delta at D + 1 - rank) is bary_r = R_{D-r} - R_{D+1-r}, bary_0 = R_D + (1 - R_0)
    float delta[D + 1], R[D + 1];
#pragma unroll
    for (int i = 0; i <= D; i++) delta[i] = __fmul_rn(__fsub_rn(e[i], (float)s.rem0[i]), kInv);
    by_rank<D>(s, delta, R);
    s.bary[0] = __fadd_rn(R[D], __fsub_rn(1.0f, R[0]));
#pragma unroll
    for (int r = 1; r <= D; r++) s.bary[r] = __fsub_rn(R[D - r], R[D + 1 - r]);
    s.bary[D + 1] = -R[0];
}
// tangent of the barycentric weights along the (scaled) direction dcf: the same rank scatter applied to its elevation
template <int D>
__device__ __forceinline__ void bary_tangent(const float* dcf, const Simplex<D>& s, float* db) {
    constexpr float kInv = 1.0f / (float)(D + 1);
    float de[D + 1], dD[D + 1], sm = 0.f;
#pragma unroll
    for (int i = D; i > 0; i--) { de[i] = (sm - (float)i * dcf[i - 1]) * kInv; sm += dcf[i - 1]; }
    de[0] = sm * kInv;
    by_rank<D>(s, de, dD);
    db[0] = dD[D] - dD[0];
#pragma unroll
    for (int r = 1; r <= D; r++) db[r] = dD[D - r] - dD[D + 1 - r];
}
// h mod T without a division: q = umulhi(h, floor(2^32 / T)) is the quotient or one less, so one conditional subtraction finishes it
// (exact for every 32-bit h; a power-of-two T needs no correction). `magic` = t_magic(T), computed on the host.
inline unsigned t_magic(int T) { return T <= 1 ? 0xffffffffu : (unsigned)(0x100000000ull / (unsigned long long)(unsigned)T); }
// The hash h = ((k0 P + k1) P + ...) P (mod 2^32) of the vertex key k_i = rem0[i] + r - (D+1) [rank[i] > D - r], i < D, is linear in the
// key over the ring Z / 2^32: h_r = h_0 + r (P^D + ... + P) - sum_i [rank[i] > D - r] (D+1) P^(D-i) with h_0 = sum_i rem0[i] P^(D-i), so the
// D+1 vertices of a simplex share h_0 (D multiply-adds) and each one costs D compare + subtract pairs -- same bits as the
// multiply chain per vertex, less than half of its instructions.
template <int D>
__device__ __forceinline__ unsigned vindex(const Simplex<D>& s, int r, unsigned magic, unsigned T) {
    constexpr unsigned P1 = 2531011u;
    unsigned pw[D];                    // pw[i] = P^(D - i)
    pw[D - 1] = P1;
#pragma unroll
    for (int i = D - 2; i >= 0; i--) pw[i] = pw[i + 1] * P1;
    unsigned h = 0u, psum = 0u;
#pragma unroll
    for (int i = 0; i < D; i++) { h += (unsigned)s.rem0[i] * pw[i]; psum += pw[i]; }
    h += (unsigned)r * psum;
#pragma unroll
    for (int i = 0; i < D; i++)
        if (s.rank[i] > D - r) h -= (unsigned)(D + 1) * pw[i];
    unsigned rem = h - __umulhi(h, magic) * T;
    return rem >= T ? rem - T : rem;
}

// exact (erf) GELU and derivatives from one exp and one reciprocal: Phi(z) by Abramowitz-Stegun 7.1.26 (|err| < 1e-7),
// whose e^{-x^2} factor at x = z / sqrt(2) is the Gaussian that the derivative needs anyway.
struct GeluEval { float cdf, pdf; };
__device__ __forceinline__ GeluEval gelu_eval(float z) {
    GeluEval o;
    float E = __expf(-0.5f * z * z);
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752f, fabsf(z), 1.0f)));
    float poly = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
    float q = 0.5f * poly * E;
    o.cdf = z >= 0.f ? 1.0f - q : q;
    o.pdf = 0.3989422804014327f * E;
    return o;
}

struct FusedParams {
    int N, L, T;
    unsigned cap_mask;   // t_magic(T): multiplier of the division-free h mod T (any capacity, not only powers of two)
    float points_scaling;
    int in_dim;          // (L + E) * 2 feature columns
    int knockout = 0;    // diagnostics only (PSDF_EXPERIMENT_KNOCKOUT, k_sdf_lattice_scatter): bit 0 issue no reduction, bit 1 no warp
                         // aggregation -- "what would this cost if it were free" timings (results are garbage); 0 in production
    MlpGeom g;
};

// ---------------------------------------------------------------------------------------------- encoder of one level (D = 3, 4; F = 2)
// Level constants in shared memory; scale / shift rows padded to 4 floats.
struct LevelC { float scale[kMaxLevels * 4]; float shift[kMaxLevels * 4]; float window[kMaxLevels]; };
template <int D = 3>
__device__ __forceinline__ void load_level_consts(LevelC* lc, int L, const float* scale, const float* shift, const float* window, int tid,
                                                  int nthreads) {
    for (int i = tid; i < L * D; i += nthreads) {
        lc->scale[(i / D) * 4 + (i % D)] = scale[i];
        lc->shift[(i / D) * 4 + (i % D)] = shift ? shift[i] : 0.0f;
    }
    for (int i = tid; i < L; i += nthreads) lc->window[i] = window ? window[i] : 1.0f;
}
// The two window-weighted features (a0, a1) = w sum_r B_r v_r of position x at level l. Also returns the simplex s and the D+1 vertex
// values v, from which the callers form tangents.
template <int D>
__device__ __forceinline__ float2 level_features(const float* x, const LevelC* lc, int l, const float2* __restrict__ lattice, int T,
                                                 unsigned cap_mask, Simplex<D>& s, float2* v) {
    float cf[D], e[D + 1];
#pragma unroll
    for (int i = 0; i < D; i++) cf[i] = __fmul_rn(__fadd_rn(x[i], lc->shift[l * 4 + i]), lc->scale[l * 4 + i]);
    elevate<D>(cf, e);
    locate<D>(e, s);
    const float w = lc->window[l];      // read before the gathers: with this order ptxas spills the least in k_sdf_fused_backward
    const float2* tab = lattice + (size_t)l * T;
#pragma unroll
    for (int r = 0; r <= D; r++) v[r] = __ldg(tab + vindex<D>(s, r, cap_mask, (unsigned)T));
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int r = 0; r <= D; r++) { const float wr = s.bary[r] * w; a0 = fmaf(v[r].x, wr, a0); a1 = fmaf(v[r].y, wr, a1); }
    return make_float2(a0, a1);
}
// d feat / d x_j (j = 0..2, the spatial coordinates) of one level's two features: ft[j] = w scale_j / (D+1) * sum_i E[i][j] G_i, with
// G_i = u_{rank_i}, u_k = d feat / d D_k (by_rank) and E the (D+1) x D elevation matrix, rows {1,1,1,..},{-1,1,1,..},{0,-2,1,..},{0,0,-3,..},..;
// E[i][j] = 0 for i > j + 1, so rows 0..3 suffice for j < 3 at any D
template <int D, int K = 0>
__device__ __forceinline__ float2 u_pick(const float2* u, int rk) {
    if constexpr (K == D) return u[D];
    else return rk == K ? u[K] : u_pick<D, K + 1>(u, rk);
}
template <int D>
__device__ __forceinline__ void spatial_tangents(const Simplex<D>& s, const float2* v, float w, const float* scale, float2* ft) {
    constexpr float kInv = 1.0f / (float)(D + 1);
    float2 G[4];
    if constexpr (D == 3) {
        float2 u[4];
        u[0] = make_float2(v[3].x - v[0].x, v[3].y - v[0].y);
        u[1] = make_float2(v[2].x - v[3].x, v[2].y - v[3].y);
        u[2] = make_float2(v[1].x - v[2].x, v[1].y - v[2].y);
        u[3] = make_float2(v[0].x - v[1].x, v[0].y - v[1].y);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int rk = s.rank[i];
            G[i].x = rk == 0 ? u[0].x : (rk == 1 ? u[1].x : (rk == 2 ? u[2].x : u[3].x));
            G[i].y = rk == 0 ? u[0].y : (rk == 1 ? u[1].y : (rk == 2 ? u[2].y : u[3].y));
        }
    } else {
        float2 u[D + 1];
        u[0] = make_float2(v[D].x - v[0].x, v[D].y - v[0].y);
#pragma unroll
        for (int k = 1; k <= D; k++) u[k] = make_float2(v[D - k].x - v[D + 1 - k].x, v[D - k].y - v[D + 1 - k].y);
#pragma unroll
        for (int i = 0; i < 4; i++) G[i] = u_pick<D>(u, s.rank[i]);
    }
    const float c0 = kInv * w * scale[0], c1 = kInv * w * scale[1], c2 = kInv * w * scale[2];
    const float s01x = G[0].x + G[1].x, s01y = G[0].y + G[1].y;
    ft[0] = make_float2(c0 * (G[0].x - G[1].x), c0 * (G[0].y - G[1].y));
    ft[1] = make_float2(c1 * fmaf(-2.0f, G[2].x, s01x), c1 * fmaf(-2.0f, G[2].y, s01y));
    ft[2] = make_float2(c2 * fmaf(-3.0f, G[3].x, s01x + G[2].x), c2 * fmaf(-3.0f, G[3].y, s01y + G[2].y));
}
// Operand core kc past the 2L lattice features: column 2L + d = x_d * points_scaling for d < D (and below in_dim), zero padding up to
// Kp[0]. With NT tangents, column 2L + d of tangent j is dx[j][d] * points_scaling for the spatial d < 3 and zero for the time column.
template <int NT, int D = 3>
__device__ __forceinline__ void concat_core(const FusedParams& P, int kc, const float* x, const float (*dx)[3], float* fv, float (*ft)[8]) {
    const int c0 = 2 * P.L;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int c = kc * 8 + i - c0;
        fv[i] = 0.f;
#pragma unroll
        for (int j = 0; j < NT; j++) ft[j][i] = 0.f;
#pragma unroll
        for (int d = 0; d < D; d++) {
            if (c == d && (c0 + c) < P.in_dim) {
                fv[i] = x[d] * P.points_scaling;
                if (d < 3) {
#pragma unroll
                    for (int j = 0; j < NT; j++) ft[j][i] = dx[j][d] * P.points_scaling;
                }
            }
        }
    }
}

// store 8 consecutive K values of one row into a hi/lo operand tile pair (one 16-byte core-matrix row each)
__device__ __forceinline__ void store8(uint8_t* a_hi, uint8_t* a_lo, int row, int kcore, const float* v) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        umma::split2_bf16(v[2 * i], v[2 * i + 1], h[i], l[i]);
    }
    int off = (row >> 3) * kSBO_A + kcore * kLBO + (row & 7) * 16;
    *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
}
// bf16 hi / lo pair of two adjacent columns of one row -> the two operand tiles (4-byte stores; a warp covers whole 128-byte cores);
// sbo: the tiles' 8-row-group stride
__device__ __forceinline__ void store_pair(uint8_t* t_hi, uint8_t* t_lo, int row, int col, float x0, float x1, int sbo = kSBO_A) {
    uint32_t h, l;
    umma::split2_bf16(x0, x1, h, l);
    const int off = (row >> 3) * sbo + (col >> 3) * kLBO + (row & 7) * 16 + (col & 7) * 2;
    *reinterpret_cast<uint32_t*>(t_hi + off) = h;
    *reinterpret_cast<uint32_t*>(t_lo + off) = l;
}
// fragment row / column of accumulator entry 4 j + 2 h + b of rows 64 mh .. 64 mh + 63 (umma::wg_mma_regs layout; warp w of the
// warpgroup, lane t)
__device__ __forceinline__ int frag_row(int mh, int h) { return 64 * mh + 16 * ((threadIdx.x >> 5) & 3) + (threadIdx.x & 31) / 4 + 8 * h; }
__device__ __forceinline__ int frag_col(int j) { return 8 * j + 2 * (threadIdx.x & 3); }
// Columns [n0, n0 + N) of D_s = A_s W^T, s = 0 .. S-1, for the 64 rows starting `row_off` bytes into the A tiles, into the issuing
// warpgroup's registers (umma::wg_mma_regs fragments): stream s lands in acc + 16 s, so the values of all streams at one (row, column)
// are in the same thread. Stream s's A tiles are a + s * stream_bytes (hi) and + lo_bytes (lo), with the 8-row-group stride a_sbo; the
// weight tile is [Np rows][Kp] K-major.
template <int N, int S>
__device__ __forceinline__ void streams_product(float* acc, const uint8_t* a, int stream_bytes, int lo_bytes, uint32_t row_off,
                                                const uint8_t* w_hi, const uint8_t* w_lo, int Kp, int n0, int a_sbo = kSBO_A) {
    static_assert(S == 1 || N <= 32, "a stream's fragment holds 16 floats");
    const uint32_t sbo_w = (Kp / 8) * kLBO, wo = (uint32_t)(n0 / 8) * sbo_w;
    const uint64_t dwh = umma::make_desc(umma::smem_u32(w_hi) + wo, kLBO, sbo_w), dwl = umma::make_desc(umma::smem_u32(w_lo) + wo, kLBO, sbo_w);
    uint64_t dah[S], dal[S];
#pragma unroll
    for (int s = 0; s < S; s++) {
        const uint8_t* as = a + s * stream_bytes;
        dah[s] = umma::make_desc(umma::smem_u32(as) + row_off, kLBO, a_sbo);
        dal[s] = umma::make_desc(umma::smem_u32(as + lo_bytes) + row_off, kLBO, a_sbo);
    }
    umma::wgmma_fence();
    umma::wg_mma_streams<N, 0, 0, S>(acc, dah, dal, dwh, dwl, (2 * kLBO) >> 4, (2 * kLBO) >> 4, Kp / 16, false);
    umma::wgmma_commit();
    umma::wgmma_wait0();
}
// The reverse product of streams_product: columns [n0, n0 + N) of D_s = A_s W, s = 0 .. S-1, the reduction running over the Np rows of
// the FORWARD weight tile [Np rows][Kp] read as an MN-major B operand (8-row groups sbo_w apart, 8-column cores kLBO apart), so no
// transposed copy is needed. A operands and fragments as in streams_product. Issue only: the caller brackets it with wgmma_fence() and
// wgmma_commit() + wgmma_wait0().
template <int N, int S>
__device__ __forceinline__ void streams_product_wt(float* acc, const uint8_t* a, int stream_bytes, int lo_bytes, uint32_t row_off,
                                                   const uint8_t* w_hi, const uint8_t* w_lo, int Kp, int Np, int n0) {
    static_assert(S == 1 || N <= 32, "a stream's fragment holds 16 floats");
    const uint32_t sbo_w = (Kp / 8) * kLBO, wo = (uint32_t)(n0 / 8) * kLBO;
    const uint64_t dwh = umma::make_desc(umma::smem_u32(w_hi) + wo, sbo_w, kLBO), dwl = umma::make_desc(umma::smem_u32(w_lo) + wo, sbo_w, kLBO);
    uint64_t dah[S], dal[S];
#pragma unroll
    for (int s = 0; s < S; s++) {
        const uint8_t* as = a + s * stream_bytes;
        dah[s] = umma::make_desc(umma::smem_u32(as) + row_off, kLBO, kSBO_A);
        dal[s] = umma::make_desc(umma::smem_u32(as + lo_bytes) + row_off, kLBO, kSBO_A);
    }
    umma::wg_mma_streams<N, 0, 1, S>(acc, dah, dal, dwh, dwl, (2 * kLBO) >> 4, (2 * sbo_w) >> 4, Np / 16, false);
}


// column halves of an N-column product in units of 16 columns (MMA N % 16 == 0); the second half may be empty
__device__ __forceinline__ void split_n(int N, int half, int& n0, int& nn) {
    const int na = ((N / 16 + 1) / 2) * 16;
    n0 = half ? na : 0;
    nn = half ? N - na : na;
}

// rows [64 mh, 64 mh + 64) of one stream of D[128 x Np] = A[128 x Kp] W^T as the three split products (one warpgroup, see
// umma::wg_gemm). A tiles have the 8-row-group stride a_sbo; the weight tile is [Np rows][Kp] K-major. Descriptor convention
// checked by tests/test_fused_gpu.py::test_umma_gemm_self_test: the first offset field (LBO) is the stride between core
// matrices adjacent along K, the second (SBO) between 8-row groups.
__device__ __forceinline__ void issue_gemm(uint32_t tmem_d, int mh, const uint8_t* a_hi, const uint8_t* a_lo, const uint8_t* w_hi,
                                           const uint8_t* w_lo, int Kp, int Np, int a_sbo = kSBO_A) {
    const uint32_t sbo_w = (Kp / 8) * kLBO;
    const uint32_t ao = (uint32_t)(mh * 8 * a_sbo);
    const uint64_t dah = umma::make_desc(umma::smem_u32(a_hi) + ao, kLBO, a_sbo), dal = umma::make_desc(umma::smem_u32(a_lo) + ao, kLBO, a_sbo);
    const uint64_t dwh = umma::make_desc(umma::smem_u32(w_hi), kLBO, sbo_w), dwl = umma::make_desc(umma::smem_u32(w_lo), kLBO, sbo_w);
    umma::wg_gemm<0, 0>(tmem_d + ((uint32_t)(64 * mh) << 16), false, dah, dal, dwh, dwl, (2 * kLBO) >> 4, (2 * kLBO) >> 4, (8 * sbo_w) >> 4,
                        Kp / 16, Np, false);
}

// v broadcast from lane 0. For values that are the same in every lane of a warp but that ptxas cannot prove so: the warp index, and
// the per-layer geometry P.g.*[l] under a runtime l (read per thread with a register index). Branches and wgmma k-loops bounded by
// such values count as divergent for ptxas, which then serializes the wgmma chains behind them (C7520: a wait after every HGMMA).
__device__ __forceinline__ int warp_uniform(int v) { return __shfl_sync(0xffffffffu, v, 0); }

// ---------------------------------------------------------------------------------------------- backward helpers
constexpr unsigned kFull = 0xffffffffu;
// Warp aggregation of the lattice scatter (match_any + segmented shuffle sum, one red per distinct vertex) pays where the 32
// neighbouring samples of a warp share vertices: on levels whose cells are larger than the sample spacing. On the fine levels
// (scale factor 1 / (sqrt(2) sigma) above this bound, i.e. sigma below ~3.5e-3) hardly any two lanes meet, so they issue their reds
// directly and skip the match.
constexpr float kAggregateBelowScale = 200.0f;
__device__ __forceinline__ float2 add_peers2(unsigned peers, float2 x, int lane) {
    // coarse levels: the 32 neighbouring samples of a warp very often all hit the same vertex -> plain butterfly (10 shuffles)
    if (__all_sync(kFull, peers == kFull)) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { x.x += __shfl_xor_sync(kFull, x.x, o); x.y += __shfl_xor_sync(kFull, x.y, o); }
        return x;
    }
    int rel = __popc(peers << (31 - lane) << 1);
    peers &= (0xfffffffeu << lane);
    while (__any_sync(kFull, peers)) {
        int next = __ffs(peers);
        float tx = __shfl_sync(kFull, x.x, (next - 1) & 31);
        float ty = __shfl_sync(kFull, x.y, (next - 1) & 31);
        if (next) { x.x += tx; x.y += ty; }
        int done = rel & 1;
        peers &= __ballot_sync(kFull, !done);
        rel >>= 1;
    }
    return x;
}
__device__ __forceinline__ void red_v2(float* addr, float2 v) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ void red_v4(float* addr, float a, float b, float c, float d) {     // 16-byte aligned address
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// one lattice-gradient contribution: float atomics, or fixed point (deterministic mode, ftab != NULL)
__device__ __forceinline__ void scatter2(float* gtab, unsigned long long* ftab, unsigned idx, float2 cv) {
    if (ftab) { fx_add(ftab + (size_t)idx * 2, cv.x); fx_add(ftab + (size_t)idx * 2 + 1, cv.y); }
    else red_v2(gtab + (size_t)idx * 2, cv);
}
// Encoder backward of one sample at one level, called by a whole warp (one sample per lane):
//     lattice[idx_r] += w (B_r abar + dB_r tabar),  r = 0..D,   abar = (a0, a1), tabar = (t0, t1) of the level's two features
// x, v: position and tangent direction (D coordinates); scale3 / shift3: the level's scale and shift; gtab / ftab: the level's float /
// fixed-point gradient table (scatter2). TAN = false: no tangent term (v, t0, t1 unused), lattice[idx_r] += w B_r abar. Invalid lanes add
// nothing. aggregate: warp-uniform, sum the lanes that share a vertex first (match_any + add_peers2, one reduction per distinct vertex);
// do_red = false issues no reduction (diagnostics, PSDF_EXPERIMENT_KNOCKOUT).
template <bool TAN, int D = 3>
__device__ __forceinline__ void scatter_level(const float* x, const float* v, const float* scale3, const float* shift3, float w, float a0,
                                              float a1, float t0, float t1, bool valid, bool aggregate, bool do_red, int lane,
                                              unsigned cap_mask, unsigned T, float* gtab, unsigned long long* ftab) {
    float cf[D], dcf[D], e[D + 1];
#pragma unroll
    for (int i = 0; i < D; i++) {
        cf[i] = __fmul_rn(__fadd_rn(x[i], shift3[i]), scale3[i]);
        if constexpr (TAN) dcf[i] = v[i] * scale3[i];
    }
    elevate<D>(cf, e);
    Simplex<D> s;
    locate<D>(e, s);
    float db[D + 2];
    if constexpr (TAN) bary_tangent<D>(dcf, s, db);
#pragma unroll
    for (int r = 0; r <= D; r++) {
        unsigned idx = vindex<D>(s, r, cap_mask, T);
        float cb = s.bary[r] * w;
        float2 cv;
        if constexpr (TAN) {
            float cd = db[r] * w;
            cv = make_float2(cb * a0 + cd * t0, cb * a1 + cd * t1);
        } else {
            cv = make_float2(cb * a0, cb * a1);
        }
        if (aggregate) {
            unsigned key = valid ? idx : 0xffffffffu;
            unsigned peers = __match_any_sync(kFull, key);
            cv = add_peers2(peers, cv, lane);
            if (valid && lane == __ffs(peers) - 1 && do_red) scatter2(gtab, ftab, idx, cv);
        } else if (valid && (do_red || cv.x == 123.456f)) {
            scatter2(gtab, ftab, idx, cv);
        }
    }
}
// column sums of 16 per-lane values over the 32 lanes of a warp with 16 shuffles (halving butterfly): afterwards both
// lanes of the pair {2p, 2p+1} hold the sum of column `col` = bit-reversal-free index built from lane bits 4..1.
__device__ __forceinline__ float colsum16(const float* v, int lane, int& col) {
    float a[8], b[4], c[2], d;
    bool up = lane & 16;
#pragma unroll
    for (int i = 0; i < 8; i++) { float send = up ? v[i] : v[i + 8], keep = up ? v[i + 8] : v[i]; a[i] = keep + __shfl_xor_sync(kFull, send, 16); }
    up = lane & 8;
#pragma unroll
    for (int i = 0; i < 4; i++) { float send = up ? a[i] : a[i + 4], keep = up ? a[i + 4] : a[i]; b[i] = keep + __shfl_xor_sync(kFull, send, 8); }
    up = lane & 4;
#pragma unroll
    for (int i = 0; i < 2; i++) { float send = up ? b[i] : b[i + 2], keep = up ? b[i + 2] : b[i]; c[i] = keep + __shfl_xor_sync(kFull, send, 4); }
    up = lane & 2;
    { float send = up ? c[0] : c[1], keep = up ? c[1] : c[0]; d = keep + __shfl_xor_sync(kFull, send, 2); }
    d += __shfl_xor_sync(kFull, d, 1);
    col = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    return d;
}
// Column sums of a fragment block over the 8 lanes t / 4 = 0..7 of one warp (halving butterfly over lanes ^ 16, ^ 8, ^ 4, 7 shuffles): v[2 j + b]
// is this thread's value of column 8 j + 2 (t % 4) + b. Afterwards every lane holds the sum of one column, `col` = 8 (2 bit4 + bit3) +
// 2 (t % 4) + bit2.
__device__ __forceinline__ float frag_colsum8(const float* v, int lane, int& col) {
    float a[4], b[2], c;
    bool up = lane & 16;
#pragma unroll
    for (int i = 0; i < 4; i++) { float send = up ? v[i] : v[i + 4], keep = up ? v[i + 4] : v[i]; a[i] = keep + __shfl_xor_sync(kFull, send, 16); }
    up = lane & 8;
#pragma unroll
    for (int i = 0; i < 2; i++) { float send = up ? a[i] : a[i + 2], keep = up ? a[i + 2] : a[i]; b[i] = keep + __shfl_xor_sync(kFull, send, 8); }
    up = lane & 4;
    { float send = up ? b[0] : b[1], keep = up ? b[1] : b[0]; c = keep + __shfl_xor_sync(kFull, send, 4); }
    col = 8 * (2 * ((lane >> 4) & 1) + ((lane >> 3) & 1)) + 2 * (lane & 3) + ((lane >> 2) & 1);
    return c;
}
// Bias-gradient column sums of an M = 64 fragment block over each 32-row group, i.e. over the warp pair 2p, 2p + 1 of a warpgroup.
// v: this thread's 16 values (v[4 j + 2 h + b], umma::wg_mma_regs layout), columns 8 j + 2 (t % 4) + b of which the first nn count (rows
// outside the problem hold 0). The rows r = 0..31 of the group are added in the order of colsum16 over one warp in the per-row layout:
// pairs r, r ^ 16 first, then r ^ 8, r ^ 4, r ^ 2, r ^ 1. Here bit 4 of r is the warp of the pair, bit 3 the fragment half h and bits 2..0
// the lane bits 4..2, so the odd warp's values come through shared memory (bx: the pair's [16][32] floats), then h, then
// frag_colsum8's butterfly. Every partial sum, and so the one fixed-point rounding per tile, column and 32 rows, is that of the per-row
// sum. Both warps of the pair call it (named barrier bar_id); true in the even warp's lanes that hold the sum `cs` of a column col < nn.
__device__ __forceinline__ bool frag_pair_colsum(const float* v, int nn, float* bx, int bar_id, float& cs, int& col) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    bx += lane;
    if (warp & 1) {
#pragma unroll
        for (int i = 0; i < 16; i++) if (2 * i < nn) bx[i * 32] = v[i];
    }
    umma::bar_sync(bar_id, 64);
    if (warp & 1) return false;
    float bs[8];
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
        for (int b = 0; b < 2; b++) {
            const int i0 = 4 * j + b, i1 = 4 * j + 2 + b;
            bs[2 * j + b] = (8 * j < nn) ? (v[i0] + bx[i0 * 32]) + (v[i1] + bx[i1 * 32]) : 0.f;
        }
    cs = frag_colsum8(bs, lane, col);
    return col < nn;
}

// Weight gradients of a persistent backward kernel whose CTAs each leave their sum of every weight in a slab of their own, with plain
// stores: slot (l, m, k) of CTA c at (c * kNL + l) * LD * LD + m * LD + k. The CTAs' values of one slot (layer blockIdx.y, row-major
// index i over the true [N_l, K_l]; Slab::get() is the slab array's device address) are added up over the CTAs of chunk blockIdx.z, then one atomic adds the partial sum. T = unsigned
// long long: fixed-point sums (fx_of), added in integer arithmetic (exact, in any order) and then into the deterministic accumulators,
// or as their float value into the gradient; T = float: float sums, added into the gradient. Flushing every CTA's sums with atomics at
// the end of the persistent kernel is bound by the L2 atomic throughput on the same few thousand addresses (one reduction per weight
// and CTA); here the sums are read once with coalesced loads and kDwReduceChunks partial sums per slot are reduced.
constexpr int kDwReduceThreads = 256, kDwReduceChunks = 4;
struct DwSums {
    float* gW[kNL];                 // [N_l, K_l] (+=)
    unsigned long long* fx_mlp;     // deterministic mode (T = unsigned long long): fixed-point accumulators, layer l at l * fx_w; else NULL
    int fx_w;
};
template <int LD, typename T, typename Slab>
static __global__ void __launch_bounds__(kDwReduceThreads) k_dw_reduce(MlpGeom g, int ctas, DwSums s) {
    const int l = blockIdx.y;
    // no dynamic indexing of the parameter struct (local-memory copy)
    const int K = l == 0 ? g.K[0] : (l == 1 ? g.K[1] : (l == 2 ? g.K[2] : g.K[3]));
    const int N = l == 0 ? g.N[0] : (l == 1 ? g.N[1] : (l == 2 ? g.N[2] : g.N[3]));
    const int i = blockIdx.x * kDwReduceThreads + threadIdx.x;
    if (i >= N * K) return;
    const int m = i / K, k = i - m * K;
    const int per = (ctas + kDwReduceChunks - 1) / kDwReduceChunks, c0 = blockIdx.z * per, c1 = min(ctas, c0 + per);
    const T* src = reinterpret_cast<const T*>(Slab::get()) + (size_t)l * LD * LD + m * LD + k;
    T v = T(0);
#pragma unroll 8
    for (int c = c0; c < c1; c++) v += src[(size_t)c * kNL * LD * LD];
    if (v == T(0)) return;
    float* gw = l == 0 ? s.gW[0] : (l == 1 ? s.gW[1] : (l == 2 ? s.gW[2] : s.gW[3]));
    if constexpr (std::is_same<T, float>::value) atomicAdd(gw + i, v);
    else if (s.fx_mlp) atomicAdd(s.fx_mlp + l * s.fx_w + i, v);
    else atomicAdd(gw + i, (float)((double)(long long)v / kFxScale));
}


}  // namespace psdf_fused
