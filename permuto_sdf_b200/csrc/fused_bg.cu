// Fused background network for sm_90a: NerfHash.forward of the reference without its colour head (permuto_sdf_py/models/models.py:425-563)
//     feat    = permutohedral_encoding(x4) (+ concat points)              2L + 4 columns (D = 4)
//     z       = trunk(feat): K0 -> 64 -> 64 -> 64 -> 65, GELU between layers
//     density = softplus(z[:, 0])
//     rgb_raw = head([gelu(z[:, 1:65]) | SH_4(view dir) (16)]): 80 -> 64 -> 64 -> 3, GELU between layers
// Seven linear layers, one CTA = one 128-sample tile per step (persistent grid), 512 threads (row = tid & 127, group = tid >> 7).
// Operand tiles, split products and weight streaming are those of the colour network (fused_rgb_common.cuh): every layer is three bf16
// hi/lo split products on wgmma, each layer's weight block arrives by one TMA bulk copy into a single buffer.
// Column layout of the activation tile: [0, Kp0) encoder | [0, 64) hidden activations | [64, 80) SH_4, written once per tile and read by
// layer 4 only. The packed trunk output layer is rotated by one row (psdf_bg_mlp_pack): columns 0..63 are the 64 colour features and
// column 64 the density, so gelu(z[:, 1:65]) is written in place as columns 0..63 of layer 4's input.
//
// Backward (k_bg_fused_backward): recompute of layers 0..5 with the pre-activations kept in the accumulator area, then the reverse sweep
// l = 6..0: abar_l = zbar^(l) W_l on the tensor cores (warpgroups 0 / 1) beside dW_l = zbar^(l)^T a_l (warpgroups 2 / 3, fixed-point sums
// per CTA as in fused_rgb_bwd.cu), zbar^(l-1) = abar_l gelu'(z^(l-1)) (softplus' for the density column), a_(l-1) rebuilt from the stored
// pre-activations (a_0 from the encoder). abar_0's lattice columns leave to the workspace; k_bg_lattice_scatter scatters them.
#include "fused_common.cuh"
#include "fused_rgb_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;
using namespace psdf_rgb;

namespace {
constexpr int kBgNL = 7;
constexpr int kBgHidden = 64, kBgFeat = 64, kBgSh = 16, kBgShCol = 64;
constexpr int kBgMaxCols = 80;                               // widest padded layer dimension
constexpr int kBgWBytes = kBgMaxCols * kBgMaxCols * 4;       // weight buffer: hi + lo of one layer
constexpr int kBgDensityCol = 64;                            // of the rotated trunk output
using BgGeom = MlpGeomN<kBgNL>;
constexpr int kAccFwdCols = kBgMaxCols;
constexpr int kAccBwdCols = 7 * kBgMaxCols;                  // z^(0..5) | abar work columns
__device__ float g_acc_bg[(size_t)kAccCtas * kTile * kAccFwdCols];
__device__ float g_acc_bg_bwd[(size_t)kAccCtas * kTile * kAccBwdCols];
constexpr int kBgDwLD = kBgMaxCols, kBgDwSlots = kTile * kBgDwLD;          // per layer: [128 rows][80 columns]
__device__ unsigned long long g_dw_bg_bwd[(size_t)kAccCtas * kBgNL * kBgDwSlots];
constexpr int kFxW = kBgMaxCols * kBgMaxCols, kFxB = kBgNL * kFxW;          // weight / bias offsets in DetBufs::rgb_mlp
static_assert(kFxB + kBgNL * kBgMaxCols <= 4 * kDetRgbW + 4 * 128, "fixed-point MLP accumulators");

struct BgParams {
    int N, L, T;
    unsigned cap_mask;
    float points_scaling;
    int in_dim;          // 2L + 4
    BgGeom g;
};

inline int make_bg_geom(int in_dim, BgGeom& g) {
    if (in_dim < 8 || pad16(in_dim) > kBgShCol) return PSDF_ERR_UNSUPPORTED;
    // layer 4 reads [64 features | SH_4], not the 65 trunk outputs
    const int K[kBgNL] = {in_dim, kBgHidden, kBgHidden, kBgHidden, kBgFeat + kBgSh, kBgHidden, kBgHidden};
    const int N[kBgNL] = {kBgHidden, kBgHidden, kBgHidden, kBgFeat + 1, kBgHidden, kBgHidden, 3};
    g = make_geom_kn<kBgNL>(K, N);
    return PSDF_OK;
}

inline int make_bg_params(BgParams& P, int N, int L, int T, float points_scaling) {
    if (N < 0 || L < 4 || L > kMaxLevels || (L % 4) != 0 || T < 1) return PSDF_ERR_UNSUPPORTED;
    P.N = N; P.L = L; P.T = T;
    P.cap_mask = t_magic(T);
    P.points_scaling = points_scaling;
    P.in_dim = 2 * L + 4;
    if (pad16(P.in_dim) > kBgShCol) return PSDF_ERR_UNSUPPORTED;
    return make_bg_geom(P.in_dim, P.g);
}

struct BgLayers { const float* W[kBgNL]; const float* B[kBgNL]; };
// packed trunk output row n = source row (n + 1) % 65: the 64 features first, the density last
__global__ void k_pack_bg(BgGeom g, BgLayers p, uint8_t* blob) {
    const int l = blockIdx.y;
    pack_layer_elem(g, l, blockIdx.x * blockDim.x + threadIdx.x, p.W[l], p.B[l], blob, l == 3 ? 1 : 0);
}

// Layer-0 operand tile of one sample row and the SH_4 columns of layer 4: thread (row, grp) builds the lattice cores grp, grp + 4, ...;
// group 0 the concat-point core, groups 1 / 2 the two SH cores, group 3 the zero padding up to Kp0. D = 3 (foreground NeRF) or 4
// (NeRF++ background): both give 2L + 4 columns, the concat core {x0, x1, x2, 0} * scaling at D = 3.
template <int D>
__device__ __forceinline__ void build_bg_input(const BgParams& P, const LevelC* lc, const float2* __restrict__ lattice,
                                               const float* __restrict__ pos, const float* __restrict__ dirs, int n, bool valid, int row,
                                               int grp, uint8_t* a_hi, uint8_t* a_lo, bool with_sh) {
    float x[4] = {0.f, 0.f, 0.f, 0.f};
    if (valid) {
#pragma unroll
        for (int i = 0; i < D; i++) x[i] = pos[(size_t)n * D + i];
    }
    const int level_cores = P.L / 4;
    for (int kc = grp; kc < level_cores; kc += kRgbGroups) {
        float fv[8];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            Simplex<D> s;
            float2 v[D + 1];
            const float2 a = level_features<D>(x, lc, kc * 4 + q, lattice, P.T, P.cap_mask, s, v);
            fv[2 * q] = a.x; fv[2 * q + 1] = a.y;
        }
        store8w(a_hi, a_lo, row, kc, fv);
    }
    if (grp == 0) {
        float t[8] = {x[0] * P.points_scaling, x[1] * P.points_scaling, x[2] * P.points_scaling, x[3] * P.points_scaling, 0.f, 0.f, 0.f, 0.f};
        store8w(a_hi, a_lo, row, level_cores, t);
    } else if (grp == 3) {
        for (int kc = level_cores + 1; kc < P.g.Kp[0] / 8; kc++) {
            float z8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            store8w(a_hi, a_lo, row, kc, z8);
        }
    } else if (with_sh) {
        float sh[kBgSh];
        float dx = 0.f, dy = 0.f, dz = 0.f;
        if (valid) { dx = dirs[(size_t)n * 3]; dy = dirs[(size_t)n * 3 + 1]; dz = dirs[(size_t)n * 3 + 2]; }
        psdf::sh_eval(dx, dy, dz, 4, sh);
        if (!valid) {
#pragma unroll
            for (int i = 0; i < kBgSh; i++) sh[i] = 0.f;
        }
        store8w(a_hi, a_lo, row, kBgShCol / 8 + grp - 1, sh + 8 * (grp - 1));
    }
}

__device__ __forceinline__ float softplus1(float z) { return z > 20.f ? z : log1pf(__expf(z)); }     // F.softplus, beta 1, threshold 20
__device__ __forceinline__ float sigmoid1(float z) { return 1.0f / (1.0f + __expf(-z)); }

// GELU of the pre-activation columns [16 c, 16 c + 16) of layer l (+ bias) -> the activation tile (the next layer's input)
__device__ __forceinline__ void gelu_chunk_to_tile(uint32_t taddr, const float* bias, uint8_t* s_a, int row, int c) {
    float z[16];
    umma::tmem_ld16(taddr, z);
#pragma unroll
    for (int i = 0; i < 16; i++) { const float zz = z[i] + bias[i]; z[i] = zz * gelu_eval(zz).cdf; }
    store8w(s_a, s_a + kWTileBytes, row, 2 * c, z);
    store8w(s_a, s_a + kWTileBytes, row, 2 * c + 1, z + 8);
}
// chunks of layer l's output that feed the next layer (the trunk output's density chunk does not)
__device__ __forceinline__ int act_chunks(const BgGeom& g, int l) { return l == 3 ? kBgFeat / 16 : g.Np[l] / 16; }

template <int D>
__global__ void __launch_bounds__(kRgbThreads, 1)
k_bg_fused(BgParams P, const float* __restrict__ pos, const float* __restrict__ dirs, const float2* __restrict__ lattice,
           const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ window, const uint8_t* __restrict__ blob,
           float* __restrict__ rgb_raw, float* __restrict__ density) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_a = smem;                                   // operand tiles [hi | lo]
    uint8_t* s_w = s_a + 2 * kWTileBytes;                  // weights of the current layer [hi | lo]
    LevelC* lc = reinterpret_cast<LevelC*>(s_w + kBgWBytes);
    float* s_bias = reinterpret_cast<float*>(lc + 1);      // 7 x 128
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_bias + kBgNL * 128);

    const int tid = threadIdx.x, warp = tid >> 5;
    const int row = tid & 127, grp = tid >> 7;
    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_fence_init();
        umma::acc_attach(g_acc_bg + (size_t)blockIdx.x * kTile * kAccFwdCols, kAccFwdCols);
    }
    load_level_consts<D>(lc, P.L, scale, shift, window, tid, kRgbThreads);
    for (int i = tid; i < kBgNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        s_bias[i] = (c < P.g.Np[l]) ? reinterpret_cast<const float*>(blob + P.g.bias[l])[c] : 0.0f;
    }
    __syncthreads();
    uint32_t w_phase = 0;
    const int ntiles = (P.N + kTile - 1) / kTile;
    if (tid == 0 && blockIdx.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int n = tile * kTile + row;
        const bool valid = n < P.N;
        build_bg_input<D>(P, lc, lattice, pos, dirs, n, valid, row, grp, s_a, s_a + kWTileBytes, true);
#pragma unroll 1
        for (int l = 0; l < kBgNL; l++) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            issue_gemm_w(0, warp >> 2, s_a, s_a + kWTileBytes, s_w, s_w + P.g.Np[l] * P.g.Kp[l] * 2, P.g.Kp[l], P.g.Np[l]);
            __syncthreads();
            if (tid == 0) {
                if (l + 1 < kBgNL) load_layer_weights(s_w, blob, P.g, l + 1, false, &bars[0]);
                else if (tile + (int)gridDim.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
            }
            const uint32_t trow = (uint32_t)((warp & 3) * 32) << 16;
            if (l < kBgNL - 1) {
                for (int c = grp; c < act_chunks(P.g, l); c += kRgbGroups) gelu_chunk_to_tile(trow + c * 16, s_bias + l * 128 + c * 16, s_a, row, c);
                if (l == 3 && grp == 0 && valid) {
                    float z[16];
                    umma::tmem_ld16(trow + kBgDensityCol, z);
                    density[n] = softplus1(z[0] + s_bias[3 * 128 + kBgDensityCol]);
                }
            } else if (grp == 0 && valid) {
                float z[16];
                umma::tmem_ld16(trow, z);
#pragma unroll
                for (int i = 0; i < 3; i++) rgb_raw[(size_t)n * 3 + i] = z[i] + s_bias[l * 128 + i];
            }
        }
        __syncthreads();      // accumulator reads / tile writes of this tile done before the next tile's encoder overwrites s_a
    }
}

struct BgBwdOut {
    float2* xch;         // [L][xch_stride] abar_0 of every level and sample slot (tile * 128 + row)
    int xch_stride;
    float* gW[kBgNL];    // [N_l, K_l] (+=)
    float* gbias[kBgNL]; // (+=)
    unsigned long long* fx_mlp;       // deterministic mode: DetBufs::rgb_mlp (layout kFxW / kFxB), else NULL
};

template <int D>
__global__ void __launch_bounds__(kRgbThreads, 1)
k_bg_fused_backward(BgParams P, const float* __restrict__ pos, const float* __restrict__ dirs, const float2* __restrict__ lattice,
                    const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ window,
                    const uint8_t* __restrict__ blob, const float* __restrict__ g_rgb, const float* __restrict__ g_density, BgBwdOut out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_a = smem;                                   // activation tiles [hi | lo]
    uint8_t* s_z = s_a + 2 * kWTileBytes;                  // adjoint tiles [hi | lo]
    uint8_t* s_w = s_z + 2 * kWTileBytes;                  // weights of the current GEMM [hi | lo]
    LevelC* lc = reinterpret_cast<LevelC*>(s_w + kBgWBytes);
    float* s_bias = reinterpret_cast<float*>(lc + 1);      // 7 x 128
    unsigned long long* s_gb = reinterpret_cast<unsigned long long*>(s_bias + kBgNL * 128);   // bias-gradient sums (float in s_gbf)
    float* s_gbf = reinterpret_cast<float*>(s_gb);
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gb + kBgNL * 128);
    const bool det = out.fx_mlp != nullptr;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row = tid & 127, grp = tid >> 7, wgi = warp >> 2;
    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_fence_init();
        umma::acc_attach(g_acc_bg_bwd + (size_t)blockIdx.x * kTile * kAccBwdCols, kAccBwdCols);
    }
    load_level_consts<D>(lc, P.L, scale, shift, window, tid, kRgbThreads);
    for (int i = tid; i < kBgNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        s_bias[i] = (c < P.g.Np[l]) ? reinterpret_cast<const float*>(blob + P.g.bias[l])[c] : 0.0f;
        s_gb[i] = 0ull;
    }
    // adjoint columns past a layer's width are read by the weight-gradient products (rows that are discarded): keep them finite
    for (int i = tid; i < 2 * kWTileBytes / 16; i += kRgbThreads) reinterpret_cast<uint4*>(s_z)[i] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    const uint32_t lane_off = (uint32_t)((warp & 3) * 32) << 16;
    auto tz = [](int l) { return (uint32_t)(l * kBgMaxCols); };
    const uint32_t t_work = (uint32_t)(6 * kBgMaxCols);
    uint32_t w_phase = 0;
    unsigned long long* dw_cta = g_dw_bg_bwd + (size_t)blockIdx.x * kBgNL * kBgDwSlots;

    const int ntiles = (P.N + kTile - 1) / kTile;
    if (tid == 0 && blockIdx.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const bool first_tile = tile == (int)blockIdx.x;
        const int n = tile * kTile + row;
        const bool valid = n < P.N;
        build_bg_input<D>(P, lc, lattice, pos, dirs, n, valid, row, grp, s_a, s_a + kWTileBytes, true);
        // ---------------- forward recompute, layers 0..5; afterwards s_a = a_6
#pragma unroll 1
        for (int l = 0; l < kBgNL - 1; l++) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            issue_gemm_w(tz(l), wgi, s_a, s_a + kWTileBytes, s_w, s_w + P.g.Np[l] * P.g.Kp[l] * 2, P.g.Kp[l], P.g.Np[l]);
            __syncthreads();
            if (tid == 0) load_layer_weights(s_w, blob, P.g, l < kBgNL - 2 ? l + 1 : kBgNL - 1, l == kBgNL - 2, &bars[0]);
            for (int c = grp; c < act_chunks(P.g, l); c += kRgbGroups)
                gelu_chunk_to_tile(tz(l) + lane_off + c * 16, s_bias + l * 128 + c * 16, s_a, row, c);
        }
        // ---------------- seed: zbar^(6) = d loss / d rgb_raw (3 of 16 columns)
        if (grp == 0) {
            float zb[16];
#pragma unroll
            for (int i = 0; i < 16; i++) zb[i] = (i < 3 && valid) ? g_rgb[(size_t)n * 3 + i] : 0.f;
            store8w(s_z, s_z + kWTileBytes, row, 0, zb);
            store8w(s_z, s_z + kWTileBytes, row, 1, zb + 8);
            int col;
            const float cs = colsum16(zb, lane, col);
            if (!(lane & 1) && col < 3) {
                if (det) fx_add(&s_gb[6 * 128 + col], cs);
                else atomicAdd(&s_gbf[6 * 128 + col], cs);
            }
        }
        // ---------------- reverse sweep l = 6..0: s_z = zbar^(l), s_a = a_l
#pragma unroll 1
        for (int l = kBgNL - 1; l >= 0; l--) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            const int Np = P.g.Np[l], Kp = P.g.Kp[l];
            if (wgi < 2) {
                // abar_l [128 x Kp] = zbar^(l) [128 x Np] W_l: B operand = W_l^T stored [Kp rows][Np]
                for (int nh = 0; nh < 2; nh++) issue_gemm_w(t_work, wgi + 2 * nh, s_z, s_z + kWTileBytes, s_w, s_w + Np * Kp * 2, Np, Kp);
            } else {
                issue_dw_w<kBgDwLD>(dw_cta + (size_t)l * kBgDwSlots, wgi - 2, s_z, s_a, Np > 64 ? 128 : 64, Kp, first_tile);
            }
            __syncthreads();
            if (tid == 0) {
                if (l > 0) load_layer_weights(s_w, blob, P.g, l - 1, true, &bars[0]);
                else if (tile + (int)gridDim.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
            }
            if (l > 0) {
                // zbar^(l-1) = abar_l gelu'(z^(l-1)) over the columns of layer l-1's output that layer l reads (+ the density column)
                const int lp = l - 1;
                for (int c = grp; c < P.g.Np[lp] / 16; c += kRgbGroups) {
                    float z[16], ab[16];
                    umma::tmem_ld16(tz(lp) + lane_off + c * 16, z);
                    umma::tmem_ld16(t_work + lane_off + c * 16, ab);
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const int col = c * 16 + i;
                        const float zz = z[i] + s_bias[lp * 128 + col];
                        if (lp == 3 && col >= kBgFeat) {
                            ab[i] = (col == kBgDensityCol && valid) ? g_density[n] * sigmoid1(zz) : 0.f;
                        } else {
                            const GeluEval ge = gelu_eval(zz);
                            ab[i] *= fmaf(zz, ge.pdf, ge.cdf);
                        }
                        if (!valid) ab[i] = 0.f;
                    }
                    store8w(s_z, s_z + kWTileBytes, row, 2 * c, ab);
                    store8w(s_z, s_z + kWTileBytes, row, 2 * c + 1, ab + 8);
                    int col;
                    const float cs = colsum16(ab, lane, col);
                    if (!(lane & 1)) {
                        if (det) fx_add(&s_gb[lp * 128 + c * 16 + col], cs);
                        else atomicAdd(&s_gbf[lp * 128 + c * 16 + col], cs);
                    }
                }
                // a_(l-1): from the stored pre-activations z^(l-2), or the encoder for a_0 (the SH columns of a_4 are still in place)
                if (lp > 0) {
                    for (int c = grp; c < act_chunks(P.g, lp - 1); c += kRgbGroups)
                        gelu_chunk_to_tile(tz(lp - 1) + lane_off + c * 16, s_bias + (lp - 1) * 128 + c * 16, s_a, row, c);
                } else {
                    build_bg_input<D>(P, lc, lattice, pos, dirs, n, valid, row, grp, s_a, s_a + kWTileBytes, false);
                }
            } else {
                // abar_0's lattice columns -> the exchange rows of k_bg_lattice_scatter
                const int slot = tile * kTile + row;
                for (int c = grp; c < (2 * P.L + 15) / 16; c += kRgbGroups) {
                    float ab[16];
                    umma::tmem_ld16(t_work + lane_off + c * 16, ab);
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        const int lv = c * 8 + q;
                        if (lv < P.L) out.xch[(size_t)lv * out.xch_stride + slot] = make_float2(ab[2 * q], ab[2 * q + 1]);
                    }
                }
            }
            __syncthreads();
        }
    }
    __syncthreads();
    // ---- this CTA's weight / bias gradients -> the deterministic accumulators (exact integer atomics) or the float gradients (+=);
    // the rotated trunk output row m is source row (m + 1) % 65
    if ((int)blockIdx.x < ntiles) {
#pragma unroll 1
        for (int l = 0; l < kBgNL; l++) {
            const int K = P.g.K[l], N = P.g.N[l];
            const unsigned long long* src = dw_cta + (size_t)l * kBgDwSlots;
            for (int i = tid; i < N * K; i += kRgbThreads) {
                const int m = i / K, k = i - m * K;
                const unsigned long long v = src[m * kBgDwLD + k];
                if (v == 0ull) continue;
                const int dst = (l == 3 ? (m + 1) % N : m) * K + k;
                if (det) atomicAdd(out.fx_mlp + l * kFxW + dst, v);
                else atomicAdd(out.gW[l] + dst, (float)((double)(long long)v / kFxScale));
            }
        }
    }
    for (int i = tid; i < kBgNL * 128; i += kRgbThreads) {
        const int l = i >> 7, c = i & 127;
        if (c >= P.g.N[l]) continue;
        const int dst = l == 3 ? (c + 1) % P.g.N[l] : c;
        if (det) { if (s_gb[i] != 0ull) atomicAdd(out.fx_mlp + kFxB + l * kBgMaxCols + dst, s_gb[i]); }
        else if (s_gbf[i] != 0.0f) atomicAdd(out.gbias[l] + dst, s_gbf[i]);
    }
}

// Encoder backward: lattice[l][idx_r] += window_l B_r abar_0[l] from the exchange rows of k_bg_fused_backward. blockIdx.y = level,
// warp = 32 consecutive sample slots. pos, scale and shift have D columns.
constexpr int kScatterThreads = 256;
template <int D>
__global__ void __launch_bounds__(kScatterThreads, 8)
k_bg_lattice_scatter(BgParams P, const float* __restrict__ pos, const float2* __restrict__ xch, int xch_stride, const float* __restrict__ scale,
                     const float* __restrict__ shift, const float* __restrict__ window, float* __restrict__ grad_lattice,
                     unsigned long long* __restrict__ fx_lattice) {
    const int slot = blockIdx.x * kScatterThreads + threadIdx.x;
    if (slot >= xch_stride) return;                                  // whole warps (xch_stride % 128 == 0)
    const int l = blockIdx.y, lane = threadIdx.x & 31;
    const bool valid = slot < P.N;
    float x[D], sc[D], sh[D];
#pragma unroll
    for (int i = 0; i < D; i++) {
        x[i] = valid ? pos[(size_t)slot * D + i] : 0.0f;
        sc[i] = scale[l * D + i];
        sh[i] = shift ? shift[l * D + i] : 0.0f;
    }
    const float w = window ? window[l] : 1.0f;
    const float2 a = xch[(size_t)l * xch_stride + slot];
    const bool aggregate = sc[0] < kAggregateBelowScale;             // warp-uniform (l is)
    scatter_level<false, D>(x, nullptr, sc, sh, w, a.x, a.y, 0.f, 0.f, valid, aggregate, true, lane, P.cap_mask, (unsigned)P.T,
                            grad_lattice + (size_t)l * P.T * 2, fx_lattice ? fx_lattice + (size_t)l * P.T * 2 : nullptr);
}

// ---------------------------------------------------------------------------------------------- NeRF compositing
// Colour head + VolumeRenderingNerf.compute_weights + integrate (permuto_sdf_py/volume_rendering/volume_rendering_modules.py:61-89) per ray:
//     c_i = sigmoid(x_i (1 + wd[img]) + b[img]),  alpha_i = 1 - exp(-sigma_i dt_i),  a_i = 1 - alpha_i + 1e-7,
//     T_i = prod_{j<i} a_j,  w_i = alpha_i T_i,  bg_rgb = sum_i w_i c_i
// One thread per ray, samples in order (the left-to-right products of the per-op path). The background (k_bg_composite*) and the
// foreground with its loss (k_nerf_loss*) share the per-sample chain below.
struct CalibArgs { const int* img; const float* wd; const float* b; int fixed; };
struct NerfAlpha { float e, alpha, a; };        // exp(-sigma dt), alpha, the factor 1 - alpha + 1e-7 of the transmittance
__device__ __forceinline__ NerfAlpha nerf_alpha(float density, float dt) {
    NerfAlpha s;
    s.e = expf(-density * dt);
    s.alpha = 1.0f - s.e;
    s.a = 1.0f - s.alpha + 1e-7f;
    return s;
}
__device__ __forceinline__ float calib_sigmoid(float x, float sc, float sh) { return 1.0f / (1.0f + expf(-(x * sc + sh))); }
__device__ __forceinline__ void calib_of(const CalibArgs& C, int ray, float* sc, float* sh, int& img) {
    img = C.img ? C.img[ray] : -1;
    const bool on = C.wd != nullptr && img != C.fixed && img >= 0;
#pragma unroll
    for (int k = 0; k < 3; k++) { sc[k] = on ? 1.0f + C.wd[img * 3 + k] : 1.0f; sh[k] = on ? C.b[img * 3 + k] : 0.0f; }
    if (!on) img = -1;
}
// per-sample colour backward: G . d c / d x_raw (=) with the calibration gradients summed over the ray
__device__ __forceinline__ float nerf_colour_backward(float G, float w, float c, float x, float sc, float& gwd, float& gb) {
    const float gz = G * w * c * (1.0f - c);            // d / d calibrated pre-activation
    gwd = fmaf(gz, x, gwd);
    gb += gz;
    return gz * sc;
}
__device__ __forceinline__ void add_calib_grads(int img, const float* gwd, const float* gb, float* g_wd, float* g_b, unsigned long long* fx) {
    if (img < 0 || !g_wd) return;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        if (fx && img < kDetImages) { fx_add(fx + img * 3 + k, gwd[k]); fx_add(fx + 3 * kDetImages + img * 3 + k, gb[k]); }
        else { atomicAdd(g_wd + img * 3 + k, gwd[k]); atomicAdd(g_b + img * 3 + k, gb[k]); }
    }
}
__global__ void __launch_bounds__(128)
k_bg_composite(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n, const float* __restrict__ x_raw,
               const float* __restrict__ density, const float* __restrict__ dt, CalibArgs C, float* __restrict__ bg_rgb) {
    const int ray = blockIdx.x * blockDim.x + threadIdx.x;
    if (ray >= nr_rays) return;
    const RayRange rr = ray_range(ray, start_end, equal, fixed_n);
    float acc[3] = {0.f, 0.f, 0.f};
    if (rr.n > 0 && rr.end <= max_nr_samples) {
        float sc[3], sh[3];
        int img;
        calib_of(C, ray, sc, sh, img);
        float T = 1.0f;
        for (int i = rr.start; i < rr.end; i++) {
            const NerfAlpha na = nerf_alpha(density[i], dt[i]);
            const float w = na.alpha * T;
#pragma unroll
            for (int k = 0; k < 3; k++) acc[k] = fmaf(w, calib_sigmoid(x_raw[(size_t)i * 3 + k], sc[k], sh[k]), acc[k]);
            T *= na.a;
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++) bg_rgb[(size_t)ray * 3 + k] = acc[k];
}
// d bg_rgb -> d x_raw [N,3], d density [N] (=) and the calibration gradients (+=; fixed point in deterministic mode)
__global__ void __launch_bounds__(128)
k_bg_composite_backward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n, const float* __restrict__ x_raw,
                        const float* __restrict__ density, const float* __restrict__ dt, CalibArgs C, const float* __restrict__ g_bg,
                        float* __restrict__ g_x, float* __restrict__ g_density, float* __restrict__ g_wd, float* __restrict__ g_b,
                        unsigned long long* __restrict__ fx) {
    const int ray = blockIdx.x * blockDim.x + threadIdx.x;
    if (ray >= nr_rays) return;
    const RayRange rr = ray_range(ray, start_end, equal, fixed_n);
    if (rr.n <= 0 || rr.end > max_nr_samples) return;
    float sc[3], sh[3], G[3], tot[3] = {0.f, 0.f, 0.f}, gwd[3] = {0.f, 0.f, 0.f}, gb[3] = {0.f, 0.f, 0.f};
    int img;
    calib_of(C, ray, sc, sh, img);
#pragma unroll
    for (int k = 0; k < 3; k++) G[k] = g_bg[(size_t)ray * 3 + k];
    // pass 1: the ray's total sum_i w_i c_i (suffix sums S_i = total - prefix_i)
    float T = 1.0f;
    for (int i = rr.start; i < rr.end; i++) {
        const NerfAlpha na = nerf_alpha(density[i], dt[i]);
        const float w = na.alpha * T;
#pragma unroll
        for (int k = 0; k < 3; k++) tot[k] = fmaf(w, calib_sigmoid(x_raw[(size_t)i * 3 + k], sc[k], sh[k]), tot[k]);
        T *= na.a;
    }
    // pass 2: d/d alpha_i = G . (T_i c_i - S_i / a_i), d alpha / d sigma = dt (1 - alpha); d/d c_i = G w_i
    T = 1.0f;
    float pre[3] = {0.f, 0.f, 0.f};
    for (int i = rr.start; i < rr.end; i++) {
        const NerfAlpha na = nerf_alpha(density[i], dt[i]);
        const float w = na.alpha * T;
        float ga = 0.f;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float x = x_raw[(size_t)i * 3 + k];
            const float c = calib_sigmoid(x, sc[k], sh[k]);
            pre[k] = fmaf(w, c, pre[k]);
            ga = fmaf(G[k], T * c - (tot[k] - pre[k]) / na.a, ga);
            g_x[(size_t)i * 3 + k] = nerf_colour_backward(G[k], w, c, x, sc[k], gwd[k], gb[k]);
        }
        g_density[i] = ga * dt[i] * na.e;
        T *= na.a;
    }
    add_calib_grads(img, gwd, gb, g_wd, g_b, fx);
}

// ---------------------------------------------------------------------------------------------- foreground NeRF compositing + loss
// train_nerf.py:67-76 + :176-182 per ray (one thread, samples left to right as in k_bg_composite):
//     w_i, c_i as above,  weights_sum = sum_i w_i,  bg_T = T of the ray's last sample (its alpha excluded; 1 for a ray without samples),
//     pred = sum_i w_i c_i + bg_T bg_rgb,
//     loss = sum_r hit_r |gt_r - pred_r|^2 / (3R) + mask_weight / R sum_r BCE(clamp(weights_sum_r, 1e-3, 1 - 1e-3), gt_mask_r)
// gt == NULL renders: no loss, pred_bg = bg_T bg_rgb.
constexpr int kNerfLossThreads = 128;
constexpr int kNerfDetSlot = 11;                 // DetBufs::loss [11, 13): the two sums in fixed point
constexpr float kBceLo = 1e-3f, kBceHi = 1.0f - 1e-3f;
struct NerfLossArgs {
    int R, max_n, fixed_n;
    const int* se;
    bool equal;
    const float* x_raw;            // [N,3]
    const float* density;          // [N]
    const float* dt;               // [N]
    CalibArgs C;
    const float* bg;               // [R,3] or NULL
    const float* gt;               // [R,3] or NULL (render)
    const uint8_t* hit;            // [R]
    const float* mask;             // [R] or NULL (no mask term)
    float mask_weight;
};
__device__ __forceinline__ float bce_term(float x, float y) {       // F.binary_cross_entropy (log clamped at -100)
    return -(y * fmaxf(logf(x), -100.0f) + (1.0f - y) * fmaxf(logf(1.0f - x), -100.0f));
}
__global__ void __launch_bounds__(kNerfLossThreads)
k_nerf_loss(NerfLossArgs A, float* __restrict__ pred, float* __restrict__ wsum_out, float* __restrict__ bgT_out, float* __restrict__ pred_bg,
            unsigned long long* fx, float* acc, float* loss, float* terms) {
    __shared__ float red[2][kNerfLossThreads / 32];
    __shared__ bool last;
    const int ray = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float v[2] = {0.f, 0.f};
    if (ray < A.R) {
        const RayRange rr = ray_range(ray, A.se, A.equal, A.fixed_n);
        float col[3] = {0.f, 0.f, 0.f}, ws = 0.f, T_last = 1.0f;
        if (rr.n > 0 && rr.end <= A.max_n) {
            float sc[3], sh[3];
            int img;
            calib_of(A.C, ray, sc, sh, img);
            float T = 1.0f;
            for (int i = rr.start; i < rr.end; i++) {
                const NerfAlpha na = nerf_alpha(A.density[i], A.dt[i]);
                const float w = na.alpha * T;
#pragma unroll
                for (int k = 0; k < 3; k++) col[k] = fmaf(w, calib_sigmoid(A.x_raw[(size_t)i * 3 + k], sc[k], sh[k]), col[k]);
                ws += w;
                T_last = T;
                T *= na.a;
            }
        }
        float p[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float b = A.bg ? __fmul_rn(T_last, A.bg[(size_t)ray * 3 + k]) : 0.0f;
            p[k] = __fadd_rn(col[k], b);
            pred[(size_t)ray * 3 + k] = p[k];
            if (pred_bg) pred_bg[(size_t)ray * 3 + k] = b;
        }
        wsum_out[ray] = ws;
        bgT_out[ray] = T_last;
        if (A.gt) {
            if (A.hit[ray]) {
#pragma unroll
                for (int k = 0; k < 3; k++) { const float d = A.gt[(size_t)ray * 3 + k] - p[k]; v[0] = fmaf(d, d, v[0]); }
            }
            if (A.mask) v[1] = bce_term(fminf(fmaxf(ws, kBceLo), kBceHi), A.mask[ray]);
        }
    }
    if (!A.gt) return;                       // render: no loss (grid-uniform)
#pragma unroll
    for (int q = 0; q < 2; q++) {
        float t = v[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) red[q][warp] = t;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        float t = 0.f;
        for (int w = 0; w < kNerfLossThreads / 32; w++) t += red[threadIdx.x][w];
        if (t != 0.0f) {
            if (fx) fx_add(fx + threadIdx.x, t);
            else atomicAdd(acc + threadIdx.x, t);
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned t = atomicAdd(reinterpret_cast<unsigned*>(acc + 2), 1u);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!last || threadIdx.x != 0) return;
    __threadfence();
    float sums[2];
    if (fx) {
        volatile unsigned long long* f = fx;
        for (int q = 0; q < 2; q++) { sums[q] = (float)((double)(long long)f[q] / kFxScale); f[q] = 0ull; }
    } else {
        volatile float* a = acc;
        for (int q = 0; q < 2; q++) sums[q] = a[q];
    }
    const float loss_rgb = sums[0] / (float)(3 * A.R), loss_mask = A.mask ? sums[1] / (float)A.R : 0.0f;
    loss[0] = loss_rgb + loss_mask * A.mask_weight;
    terms[0] = loss_rgb;
    terms[1] = loss_mask;
    for (int q = 0; q < 3; q++) acc[q] = 0.0f;        // ticket (acc[2], as bits) included: ready for the next launch
}
// d loss -> d x_raw [N,3], d density [N] (=, rows of the rays), d bg_rgb [R,3] (=) and the calibration gradients (+=):
//     G = 2 (pred - gt) hit / (3R),  g_ws = mask_weight / R * (x - y) / max(x (1 - x), 1e-12) where 1e-3 <= x = weights_sum <= 1 - 1e-3,
//     g_bgT = G . bg_rgb,  d / d alpha_i = G . (T_i c_i - S_i / a_i) + g_ws (T_i - Sw_i / a_i) - [i < n - 1] g_bgT bg_T / a_i
__global__ void __launch_bounds__(kNerfLossThreads)
k_nerf_loss_backward(NerfLossArgs A, const float* __restrict__ pred, const float* __restrict__ wsum, const float* __restrict__ bgT,
                     float* __restrict__ g_x, float* __restrict__ g_density, float* __restrict__ g_bg, float* __restrict__ g_wd,
                     float* __restrict__ g_b, unsigned long long* __restrict__ fx) {
    const int ray = blockIdx.x * blockDim.x + threadIdx.x;
    if (ray >= A.R) return;
    const float c_rgb = 2.0f / (float)(3 * A.R);
    float G[3];
#pragma unroll
    for (int k = 0; k < 3; k++) G[k] = A.hit[ray] ? c_rgb * (pred[(size_t)ray * 3 + k] - A.gt[(size_t)ray * 3 + k]) : 0.0f;
    float g_ws = 0.0f;
    if (A.mask) {
        const float x = wsum[ray];
        if (x >= kBceLo && x <= kBceHi) g_ws = A.mask_weight / (float)A.R * (x - A.mask[ray]) / fmaxf((1.0f - x) * x, 1e-12f);
    }
    const float bt = bgT[ray];
    float g_bt = 0.0f;
    if (A.bg) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float b = A.bg[(size_t)ray * 3 + k];
            g_bg[(size_t)ray * 3 + k] = G[k] * bt;
            g_bt = fmaf(G[k], b, g_bt);
        }
    }
    const RayRange rr = ray_range(ray, A.se, A.equal, A.fixed_n);
    if (rr.n <= 0 || rr.end > A.max_n) return;
    float sc[3], sh[3], tot[3] = {0.f, 0.f, 0.f}, gwd[3] = {0.f, 0.f, 0.f}, gb[3] = {0.f, 0.f, 0.f}, totw = 0.f;
    int img;
    calib_of(A.C, ray, sc, sh, img);
    float T = 1.0f;
    for (int i = rr.start; i < rr.end; i++) {
        const NerfAlpha na = nerf_alpha(A.density[i], A.dt[i]);
        const float w = na.alpha * T;
#pragma unroll
        for (int k = 0; k < 3; k++) tot[k] = fmaf(w, calib_sigmoid(A.x_raw[(size_t)i * 3 + k], sc[k], sh[k]), tot[k]);
        totw += w;
        T *= na.a;
    }
    T = 1.0f;
    float pre[3] = {0.f, 0.f, 0.f}, prew = 0.f;
    const float gb_last = g_bt * bt;
    for (int i = rr.start; i < rr.end; i++) {
        const NerfAlpha na = nerf_alpha(A.density[i], A.dt[i]);
        const float w = na.alpha * T;
        prew += w;
        float ga = g_ws * (T - (totw - prew) / na.a);
        if (i < rr.end - 1) ga -= gb_last / na.a;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float x = A.x_raw[(size_t)i * 3 + k];
            const float c = calib_sigmoid(x, sc[k], sh[k]);
            pre[k] = fmaf(w, c, pre[k]);
            ga = fmaf(G[k], T * c - (tot[k] - pre[k]) / na.a, ga);
            g_x[(size_t)i * 3 + k] = nerf_colour_backward(G[k], w, c, x, sc[k], gwd[k], gb[k]);
        }
        g_density[i] = ga * A.dt[i] * na.e;
        T *= na.a;
    }
    add_calib_grads(img, gwd, gb, g_wd, g_b, fx);
}

int persistent_grid(int ntiles) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return min(min(ntiles, sms), kAccCtas);
}

#define ST ((cudaStream_t)stream)

template <int D>
int nerf_fused_forward(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                       const float* shift, const float* window, float points_scaling, const uint8_t* blob, float* rgb_raw, float* density,
                       void* stream) {
    BgParams P;
    int rc = make_bg_params(P, N, L, T, points_scaling);
    if (rc != PSDF_OK) return rc;
    if (N == 0) return PSDF_OK;
    const size_t smem = (size_t)2 * kWTileBytes + kBgWBytes + sizeof(LevelC) + kBgNL * 128 * sizeof(float) + 64;
    { static bool optin_[64]; psdf::psdf_optin_smem(k_bg_fused<D>, 227 * 1024, optin_); }
    k_bg_fused<D><<<persistent_grid(div_up(N, kTile)), kRgbThreads, smem, ST>>>(P, pos, dirs, reinterpret_cast<const float2*>(lattice),
                                                                               scale_factor, shift, window, blob, rgb_raw, density);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

template <int D>
int nerf_fused_backward(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                        const float* shift, const float* window, float points_scaling, const uint8_t* blob, const float* g_rgb_raw,
                        const float* g_density, float* grad_lattice, uint8_t* workspace, float* const* gw, float* const* gb, void* stream) {
    BgParams P;
    int rc = make_bg_params(P, N, L, T, points_scaling);
    if (rc != PSDF_OK) return rc;
    if (N == 0) return PSDF_OK;
    const DetBufs* dbuf = det_buffers();
    if (dbuf && (long long)L * T * 2 > dbuf->lattice_len) return PSDF_ERR_UNSUPPORTED;   // reserve more with psdf_set_deterministic
    BgBwdOut out;
    for (int l = 0; l < kBgNL; l++) { out.gW[l] = gw[l]; out.gbias[l] = gb[l]; }
    out.fx_mlp = dbuf ? dbuf->rgb_mlp : nullptr;
    const int ntiles = div_up(N, kTile);
    out.xch = reinterpret_cast<float2*>(workspace);
    out.xch_stride = ntiles * kTile;
    const size_t smem = (size_t)4 * kWTileBytes + kBgWBytes + sizeof(LevelC) + kBgNL * 128 * (sizeof(float) + sizeof(unsigned long long)) + 64;
    { static bool optin_[64]; psdf::psdf_optin_smem(k_bg_fused_backward<D>, 227 * 1024, optin_); }
    k_bg_fused_backward<D><<<persistent_grid(ntiles), kRgbThreads, smem, ST>>>(P, pos, dirs, reinterpret_cast<const float2*>(lattice),
                                                                              scale_factor, shift, window, blob, g_rgb_raw, g_density, out);
    PSDF_CHECK_LAUNCH();
    k_bg_lattice_scatter<D><<<dim3(div_up(out.xch_stride, kScatterThreads), L), kScatterThreads, 0, ST>>>(
        P, pos, out.xch, out.xch_stride, scale_factor, shift, window, grad_lattice, dbuf ? dbuf->rgb_lattice : nullptr);
    PSDF_CHECK_LAUNCH();
    if (dbuf) {      // deterministic mode: fixed-point totals -> the float gradients (+=), 15 segments in two flushes
        FxSegs F, Fb;
        F.add(dbuf->rgb_lattice, grad_lattice, (long long)L * T * 2);
        for (int l = 0; l < kBgNL; l++) {
            F.add(dbuf->rgb_mlp + l * kFxW, gw[l], (long long)P.g.N[l] * P.g.K[l]);
            Fb.add(dbuf->rgb_mlp + kFxB + l * kBgMaxCols, gb[l], P.g.N[l]);
        }
        if (fx_flush(F, ST) != 0 || fx_flush(Fb, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    return PSDF_OK;
}
// the rows of N samples of pos_dim coordinates: 32-bit row and tile indexing
inline bool nerf_rows_ok(int pos_dim, int N) { return (long long)N * pos_dim <= 0x7fffffffLL && (long long)N + kTile <= 0x7fffffffLL; }

inline NerfLossArgs make_nerf_loss_args(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x_raw,
                                        const float* density, const float* dt, const int* img_idx, const float* weight_delta,
                                        const float* bias, int fixed_img, const float* bg_rgb, const float* gt_rgb, const uint8_t* hit,
                                        const float* gt_mask, float mask_weight) {
    NerfLossArgs A;
    A.R = nr_rays; A.max_n = max_nr_samples; A.se = ray_start_end; A.equal = equal != 0; A.fixed_n = fixed_n;
    A.x_raw = x_raw; A.density = density; A.dt = dt;
    A.C = {weight_delta ? img_idx : nullptr, weight_delta, bias, fixed_img};
    A.bg = bg_rgb; A.gt = gt_rgb; A.hit = hit; A.mask = gt_mask; A.mask_weight = mask_weight;
    return A;
}

}  // namespace

extern "C" {

long long psdf_bg_mlp_blob_bytes(int in_dim) {
    BgGeom g;
    if (make_bg_geom(in_dim, g) != PSDF_OK) return 0;
    return (long long)g.total + g.total_t;
}

int psdf_bg_mlp_pack(int in_dim, const float* W0, const float* b0, const float* W1, const float* b1, const float* W2, const float* b2,
                     const float* W3, const float* b3, const float* W4, const float* b4, const float* W5, const float* b5, const float* W6,
                     const float* b6, uint8_t* blob, void* stream) {
    BgGeom g;
    if (make_bg_geom(in_dim, g) != PSDF_OK) return PSDF_ERR_UNSUPPORTED;
    const BgLayers p = {{W0, W1, W2, W3, W4, W5, W6}, {b0, b1, b2, b3, b4, b5, b6}};
    dim3 grid(div_up(kBgMaxCols * kBgMaxCols, 256), kBgNL);
    k_pack_bg<<<grid, 256, 0, ST>>>(g, p, blob);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_bg_fused_forward(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                          const float* shift, const float* window, float points_scaling, const uint8_t* blob, float* rgb_raw, float* density,
                          void* stream) {
    return nerf_fused_forward<4>(N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, blob, rgb_raw, density, stream);
}

int psdf_nerf_fused_forward(int pos_dim, int N, int L, int T, const float* pos, const float* dirs, const float* lattice,
                            const float* scale_factor, const float* shift, const float* window, float points_scaling, const uint8_t* blob,
                            float* rgb_raw, float* density, void* stream) {
    if (pos_dim != 3 && pos_dim != 4) return PSDF_ERR_UNSUPPORTED;
    if (N < 0 || !nerf_rows_ok(pos_dim, N)) return PSDF_ERR_UNSUPPORTED;
    return pos_dim == 3 ? nerf_fused_forward<3>(N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, blob, rgb_raw, density, stream)
                        : nerf_fused_forward<4>(N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, blob, rgb_raw, density, stream);
}

// workspace: abar_0 of every level and sample slot (8 bytes each), sized for kMaxLevels so that the size depends on the sample count alone
long long psdf_bg_fused_backward_workspace_bytes(int N) {
    const int ntiles = div_up(N > 0 ? N : 1, kTile);
    return (long long)ntiles * kTile * kMaxLevels * (long long)sizeof(float2);
}

int psdf_bg_fused_backward(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                           const float* shift, const float* window, float points_scaling, const uint8_t* blob, const float* g_rgb_raw,
                           const float* g_density, float* grad_lattice, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3,
                           float* gW4, float* gW5, float* gW6, float* gb0, float* gb1, float* gb2, float* gb3, float* gb4, float* gb5,
                           float* gb6, void* stream) {
    float* gw[kBgNL] = {gW0, gW1, gW2, gW3, gW4, gW5, gW6};
    float* gb[kBgNL] = {gb0, gb1, gb2, gb3, gb4, gb5, gb6};
    return nerf_fused_backward<4>(N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, blob, g_rgb_raw, g_density,
                                  grad_lattice, workspace, gw, gb, stream);
}

int psdf_nerf_fused_backward(int pos_dim, int N, int L, int T, const float* pos, const float* dirs, const float* lattice,
                             const float* scale_factor, const float* shift, const float* window, float points_scaling, const uint8_t* blob,
                             const float* g_rgb_raw, const float* g_density, float* grad_lattice, uint8_t* workspace, float* gW0, float* gW1,
                             float* gW2, float* gW3, float* gW4, float* gW5, float* gW6, float* gb0, float* gb1, float* gb2, float* gb3,
                             float* gb4, float* gb5, float* gb6, void* stream) {
    if (pos_dim != 3 && pos_dim != 4) return PSDF_ERR_UNSUPPORTED;
    if (N < 0 || !nerf_rows_ok(pos_dim, N)) return PSDF_ERR_UNSUPPORTED;
    float* gw[kBgNL] = {gW0, gW1, gW2, gW3, gW4, gW5, gW6};
    float* gb[kBgNL] = {gb0, gb1, gb2, gb3, gb4, gb5, gb6};
    return pos_dim == 3 ? nerf_fused_backward<3>(N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, blob, g_rgb_raw,
                                                 g_density, grad_lattice, workspace, gw, gb, stream)
                        : nerf_fused_backward<4>(N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, blob, g_rgb_raw,
                                                 g_density, grad_lattice, workspace, gw, gb, stream);
}

int psdf_nerf_bg_composite_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x_raw,
                                   const float* density, const float* dt, const int* img_idx, const float* weight_delta, const float* bias,
                                   int fixed_img, float* bg_rgb, void* stream) {
    if (nr_rays < 0) return PSDF_ERR_ARG;
    if (nr_rays == 0) return PSDF_OK;
    const CalibArgs C = {weight_delta ? img_idx : nullptr, weight_delta, bias, fixed_img};
    k_bg_composite<<<div_up(nr_rays, 128), 128, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n, x_raw, density, dt, C, bg_rgb);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_nerf_bg_composite_backward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x_raw,
                                    const float* density, const float* dt, const int* img_idx, const float* weight_delta, const float* bias,
                                    int fixed_img, const float* g_bg_rgb, float* g_x, float* g_density, float* g_weight_delta, float* g_bias,
                                    void* stream) {
    if (nr_rays < 0) return PSDF_ERR_ARG;
    if (nr_rays == 0) return PSDF_OK;
    const CalibArgs C = {weight_delta ? img_idx : nullptr, weight_delta, bias, fixed_img};
    const DetBufs* dbuf = det_buffers();
    unsigned long long* fx = (dbuf && g_weight_delta) ? dbuf->neus : nullptr;
    k_bg_composite_backward<<<div_up(nr_rays, 128), 128, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n, x_raw, density, dt,
                                                                  C, g_bg_rgb, g_x, g_density, g_weight_delta, g_bias, fx);
    PSDF_CHECK_LAUNCH();
    if (fx) {        // deterministic mode: fixed-point calibration totals -> the float gradients (+=)
        FxSegs F;
        F.add(dbuf->neus, g_weight_delta, 3 * kDetImages);
        F.add(dbuf->neus + 3 * kDetImages, g_bias, 3 * kDetImages);
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    return PSDF_OK;
}

int psdf_nerf_loss_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x_raw,
                           const float* density, const float* dt, const int* img_idx, const float* weight_delta, const float* bias,
                           int fixed_img, const float* bg_rgb, const float* gt_rgb, const uint8_t* hit, const float* gt_mask, float mask_weight,
                           float* pred_rgb, float* weights_sum, float* bg_transmittance, float* pred_rgb_bg, float* acc, float* loss,
                           float* terms, void* stream) {
    if (nr_rays < 0 || !pred_rgb || !weights_sum || !bg_transmittance) return PSDF_ERR_ARG;
    if (gt_rgb && (!hit || !acc || !loss || !terms)) return PSDF_ERR_ARG;
    if (pred_rgb_bg && !bg_rgb) return PSDF_ERR_ARG;
    if ((long long)nr_rays * 3 > 0x7fffffffLL) return PSDF_ERR_UNSUPPORTED;
    if (nr_rays == 0) return gt_rgb ? PSDF_ERR_ARG : PSDF_OK;         // the mean over no rays is NaN in the reference
    const NerfLossArgs A = make_nerf_loss_args(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, x_raw, density, dt, img_idx, weight_delta,
                                               bias, fixed_img, bg_rgb, gt_rgb, hit, gt_mask, mask_weight);
    const DetBufs* dbuf = det_buffers();
    k_nerf_loss<<<div_up(nr_rays, kNerfLossThreads), kNerfLossThreads, 0, ST>>>(A, pred_rgb, weights_sum, bg_transmittance, pred_rgb_bg,
                                                                                dbuf ? dbuf->loss + kNerfDetSlot : nullptr, acc, loss, terms);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_nerf_loss_backward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x_raw,
                            const float* density, const float* dt, const int* img_idx, const float* weight_delta, const float* bias,
                            int fixed_img, const float* bg_rgb, const float* gt_rgb, const uint8_t* hit, const float* gt_mask,
                            float mask_weight, const float* pred_rgb, const float* weights_sum, const float* bg_transmittance, float* g_x,
                            float* g_density, float* g_bg_rgb, float* g_weight_delta, float* g_bias, void* stream) {
    if (nr_rays < 1 || !gt_rgb || !hit || !pred_rgb || !weights_sum || !bg_transmittance || !g_x || !g_density) return PSDF_ERR_ARG;
    if (bg_rgb && !g_bg_rgb) return PSDF_ERR_ARG;
    if ((long long)nr_rays * 3 > 0x7fffffffLL) return PSDF_ERR_UNSUPPORTED;
    const NerfLossArgs A = make_nerf_loss_args(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, x_raw, density, dt, img_idx, weight_delta,
                                               bias, fixed_img, bg_rgb, gt_rgb, hit, gt_mask, mask_weight);
    const DetBufs* dbuf = det_buffers();
    unsigned long long* fx = (dbuf && g_weight_delta) ? dbuf->neus : nullptr;
    k_nerf_loss_backward<<<div_up(nr_rays, kNerfLossThreads), kNerfLossThreads, 0, ST>>>(A, pred_rgb, weights_sum, bg_transmittance, g_x,
                                                                                         g_density, g_bg_rgb, g_weight_delta, g_bias, fx);
    PSDF_CHECK_LAUNCH();
    if (fx) {        // deterministic mode: fixed-point calibration totals -> the float gradients (+=)
        FxSegs F;
        F.add(dbuf->neus, g_weight_delta, 3 * kDetImages);
        F.add(dbuf->neus + 3 * kDetImages, g_bias, 3 * kDetImages);
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    return PSDF_OK;
}

}  // extern "C"
