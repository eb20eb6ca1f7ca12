// Shared pieces of the fused encoding + MLP kernels (fused_sdf.cu: forward / inference, fused_sdf_bwd.cu: training
// backward): MLP operand-blob geometry, permutohedral simplex helpers for D = 3, GELU and its derivatives, operand
// tile stores (bf16 hi/lo split in the core-matrix operand layout) and the split-product GEMM issue.
#pragma once
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

struct MlpGeom {
    int K[kNL], N[kNL];        // true dims
    int Kp[kNL], Np[kNL];      // padded dims (K % 16 == 0, N % 16 == 0)
    int w_hi[kNL], w_lo[kNL], bias[kNL];   // byte offsets in the forward blob [0, total)
    int total;
    int t_hi[kNL], t_lo[kNL];  // byte offsets of the transposed weights W_l^T ([Kp rows][Np cols]) in [total, total + total_t)
    int total_t;
};
__host__ __device__ inline int pad16(int v) { return (v + 15) & ~15; }
inline MlpGeom make_geom_dims(const int* dims) {
    MlpGeom g;
    int off = 0;
    for (int l = 0; l < kNL; l++) {
        g.K[l] = dims[l]; g.N[l] = dims[l + 1];
        g.Kp[l] = pad16(dims[l]); g.Np[l] = pad16(dims[l + 1]);
        int wbytes = g.Np[l] * g.Kp[l] * 2;
        g.w_hi[l] = off; off += wbytes;
        g.w_lo[l] = off; off += wbytes;
        g.bias[l] = off; off += g.Np[l] * 4;
    }
    g.total = (off + 127) & ~127;
    off = 0;
    for (int l = 0; l < kNL; l++) {
        int wbytes = g.Np[l] * g.Kp[l] * 2;
        g.t_hi[l] = off; off += wbytes;
        g.t_lo[l] = off; off += wbytes;
    }
    g.total_t = (off + 127) & ~127;
    return g;
}
inline MlpGeom make_geom(int in_dim, int hidden, int out_dim) {
    int dims[kNL + 1] = {in_dim, hidden, hidden, hidden, out_dim};
    return make_geom_dims(dims);
}

// weights [N][K] fp32 (torch.nn.Linear layout) -> hi/lo bf16 in the K-major core-matrix operand layout + fp32 bias;
// second half of the blob: the same weights transposed (rows = input features, K = output features) for the
// backward GEMMs dA = dZ * W
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
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    int total = g.Np[l] * g.Kp[l];
    if (e < total) {
        int n = e / g.Kp[l], k = e - n * g.Kp[l];
        float v = (n < g.N[l] && k < g.K[l]) ? W[l][n * g.K[l] + k] : 0.0f;
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
    if (e < g.Np[l]) reinterpret_cast<float*>(blob + g.bias[l])[e] = (e < g.N[l]) ? B[l][e] : 0.0f;
}

// ---------------------------------------------------------------------------------------------- lattice helpers (D = 3)
struct Simplex3 { int rem0[4]; int rank[4]; float bary[5]; };
__device__ __forceinline__ void elevate3(const float* cf, float* e) {
    float sm = 0.0f;
#pragma unroll
    for (int i = 3; i > 0; i--) { e[i] = __fmaf_rn(-(float)i, cf[i - 1], sm); sm = __fadd_rn(sm, cf[i - 1]); }
    e[0] = sm;
}
// D[k] = d[i] of the coordinate i whose rank is k (ranks are a permutation of 0..3)
__device__ __forceinline__ void by_rank(const Simplex3& s, const float* d, float* D) {
#pragma unroll
    for (int k = 0; k < 4; k++) D[k] = s.rank[0] == k ? d[0] : (s.rank[1] == k ? d[1] : (s.rank[2] == k ? d[2] : d[3]));
}
__device__ __forceinline__ void locate3(const float* e, Simplex3& s) {
    int sum = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        float v = __fmul_rn(e[i], 0.25f);
        // ceil(v) * 4 == floor(v) * 4 + 4 unless v is an integer, where both candidates coincide with e[i] and `down` wins either way
        const float down = __fmul_rn(floorf(v), 4.0f), up = __fadd_rn(down, 4.0f);
        s.rem0[i] = (__fsub_rn(up, e[i]) < __fsub_rn(e[i], down)) ? (int)up : (int)down;
        sum += s.rem0[i];
        s.rank[i] = 0;
    }
    sum /= 4;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        float di = __fsub_rn(e[i], (float)s.rem0[i]);
#pragma unroll
        for (int j = i + 1; j < 4; j++) { if (di < __fsub_rn(e[j], (float)s.rem0[j])) s.rank[i]++; else s.rank[j]++; }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        s.rank[i] += sum;
        if (s.rank[i] < 0) { s.rank[i] += 4; s.rem0[i] += 4; }
        else if (s.rank[i] > 3) { s.rank[i] -= 4; s.rem0[i] -= 4; }
    }
    // barycentric weights: with D_k the fractional offset of the coordinate of rank k, the reference's scatter
    // (+delta at 3 - rank, -delta at 4 - rank) is bary_r = D_{3-r} - D_{4-r}, bary_0 = D_3 + (1 - D_0)
    float delta[4], D[4];
#pragma unroll
    for (int i = 0; i < 4; i++) delta[i] = __fmul_rn(__fsub_rn(e[i], (float)s.rem0[i]), 0.25f);
    by_rank(s, delta, D);
    s.bary[0] = __fadd_rn(D[3], __fsub_rn(1.0f, D[0]));
    s.bary[1] = __fsub_rn(D[2], D[3]);
    s.bary[2] = __fsub_rn(D[1], D[2]);
    s.bary[3] = __fsub_rn(D[0], D[1]);
    s.bary[4] = -D[0];
}
// tangent of the barycentric weights along the (scaled) direction dcf: the same rank scatter applied to its elevation
__device__ __forceinline__ void bary_tangent3(const float* dcf, const Simplex3& s, float* db) {
    float de[4], dD[4], sm = 0.f;
#pragma unroll
    for (int i = 3; i > 0; i--) { de[i] = (sm - (float)i * dcf[i - 1]) * 0.25f; sm += dcf[i - 1]; }
    de[0] = sm * 0.25f;
    by_rank(s, de, dD);
    db[0] = dD[3] - dD[0]; db[1] = dD[2] - dD[3]; db[2] = dD[1] - dD[2]; db[3] = dD[0] - dD[1];
}
// h mod T without a division: q = umulhi(h, floor(2^32 / T)) is the quotient or one less, so one conditional subtraction finishes it
// (exact for every 32-bit h; a power-of-two T needs no correction). `magic` = t_magic(T), computed on the host.
inline unsigned t_magic(int T) { return T <= 1 ? 0xffffffffu : (unsigned)(0x100000000ull / (unsigned long long)(unsigned)T); }
// The hash h = ((k0 P + k1) P + k2) P (mod 2^32) of the vertex key k_i = rem0[i] + r - 4 [rank[i] > 3 - r] is linear in the key over the
// ring Z / 2^32: h_r = h_0 + r (P^3 + P^2 + P) - sum_i [rank[i] > 3 - r] 4 P^(3-i) with h_0 = rem0[0] P^3 + rem0[1] P^2 + rem0[2] P, so the
// four vertices of a simplex share h_0 (3 multiply-adds) and each one costs 3 compare + subtract pairs -- same bits as the
// multiply chain per vertex, less than half of its instructions.
__device__ __forceinline__ unsigned vindex3(const Simplex3& s, int r, unsigned magic, unsigned T) {
    constexpr unsigned P1 = 2531011u, P2 = P1 * P1, P3 = P2 * P1;
    unsigned h = (unsigned)s.rem0[0] * P3 + (unsigned)s.rem0[1] * P2 + (unsigned)s.rem0[2] * P1 + (unsigned)r * (P3 + P2 + P1);
    if (s.rank[0] > 3 - r) h -= 4u * P3;
    if (s.rank[1] > 3 - r) h -= 4u * P2;
    if (s.rank[2] > 3 - r) h -= 4u * P1;
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
    int free_levels = 0; // diagnostics only (PSDF_EXPERIMENT_FREE_LEVELS): the gathers of levels < free_levels read nothing (upper bound of
                         // what staging those levels' table entries in shared memory could save); 0 in production
    int skew = 1;        // k_sdf_fused_dual: group 1 starts half a sub-tile after group 0 (PSDF_SDF_FWD_SKEW=0 disables, A/B measurements)
    int knockout = 0;    // diagnostics only (PSDF_EXPERIMENT_KNOCKOUT, k_sdf_fused<true>): bit 0 skip the encoder, bit 1 issue no MMA, bit 2 skip
                         // the GELU arithmetic, bit 3 skip the operand-tile stores of the epilogue -- "what would this phase cost if it were
                         // free" timings (results are garbage); 0 in production
    MlpGeom g;
};

struct LevelC { float scale[kMaxLevels * 4]; float shift[kMaxLevels * 4]; float window[kMaxLevels]; };

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


}  // namespace psdf_fused
