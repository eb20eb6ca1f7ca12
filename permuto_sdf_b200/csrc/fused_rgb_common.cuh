// Shared pieces of the fused colour-network kernels (fused_rgb.cu forward, fused_rgb_bwd.cu backward).
// Operand tiles here are [128 samples x up to 128 columns] bf16 in the K-major core-matrix layout:
//     offset(row, col) = (row / 8) * 2048 + (col / 8) * 128 + (row % 8) * 16 + (col % 8) * 2
// Input column order of layer 0 (= torch.cat in RGB.forward, models.py:395-404), with E = 2L + 4 encoder columns:
//     [0, 2L)          lattice features, level l at columns 2l, 2l+1
//     [2L, 2L+3), 2L+3 concat points (x * scaling), zero pad
//     [E, E+25)        real spherical harmonics of degree 5 of the view direction
//     [E+25, E+28)     normalised sdf gradient
//     [E+28, E+28+G)   geometric feature (G = 32)
#pragma once
#include "fused_common.cuh"
#include "sh.cuh"

namespace psdf_rgb {
using namespace psdf_fused;

constexpr int kRgbThreads = 512;
constexpr int kRgbGroups = kRgbThreads / kTile;      // 4 threads per sample
constexpr int kWSBO = 2048;                          // 8-row-group stride of a 128-column tile
constexpr int kWTileBytes = 128 * 128 * 2;           // one bf16 tile (hi or lo)
constexpr int kGeomDim = 32;
constexpr int kShCols = 25;

struct RgbParams {
    int N, L, T;
    unsigned cap_mask;
    float points_scaling;
    int enc_cols;        // 2L + 4
    int in_dim;          // enc_cols + 25 + 3 + 32
    int acc_sdf_grad = 0; // backward: g_sdf_grad += instead of = (the caller's buffer already holds the compositing / curvature terms)
    MlpGeom g;
};

inline int make_rgb_params(RgbParams& P, int N, int L, int T, int geom_dim, float points_scaling, int h1, int h2, int h3) {
    if (N < 0 || L < 4 || L > kMaxLevels || (L % 4) != 0 || geom_dim != kGeomDim) return -3;
    P.N = N; P.L = L; P.T = T;
    P.cap_mask = t_magic(T);
    P.points_scaling = points_scaling;
    P.enc_cols = 2 * L + 4;
    P.in_dim = P.enc_cols + kShCols + 3 + kGeomDim;
    if (P.in_dim > 128 || h1 > 128 || h2 > 128 || h3 > 128 || (h1 % 16) || (h2 % 16) || (h3 % 16)) return -3;
    int dims[kNL + 1] = {P.in_dim, h1, h2, h3, 3};
    P.g = make_geom_dims(dims);
    return 0;
}

// hi + lo block of one layer (adjacent in the blob) -> the weight buffer, one TMA bulk copy (single thread)
template <int NL>
__device__ __forceinline__ void load_layer_weights(uint8_t* s_w, const uint8_t* blob, const MlpGeomN<NL>& g, int l, bool transposed, uint64_t* bar) {
    const uint32_t bytes = (uint32_t)(g.Np[l] * g.Kp[l] * 4);
    const uint8_t* src = transposed ? blob + g.total + g.t_hi[l] : blob + g.w_hi[l];
    umma::mbar_expect_tx(bar, bytes);
    umma::bulk_g2s(s_w, src, bytes, bar);
}

__device__ __forceinline__ void store8w(uint8_t* a_hi, uint8_t* a_lo, int row, int kcore, const float* v) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; i++) umma::split2_bf16(v[2 * i], v[2 * i + 1], h[i], l[i]);
    const int off = (row >> 3) * kWSBO + kcore * kLBO + (row & 7) * 16;
    *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

// quarter `part` (row half part & 1, column half part >> 1) of the three split products of [128 x Kp] x [Np x Kp]^T into the
// accumulator columns of tmem_d (one warpgroup); A tiles use the 2048-byte row-group stride
__device__ __forceinline__ void issue_gemm_w(uint32_t tmem_d, int part, const uint8_t* a_hi, const uint8_t* a_lo, const uint8_t* w_hi,
                                             const uint8_t* w_lo, int Kp, int Np) {
    int n0, nn;
    split_n(Np, part >> 1, n0, nn);
    if (nn <= 0) return;
    const int mh = part & 1;
    const uint32_t sbo_w = (Kp / 8) * kLBO;
    const uint32_t ao = (uint32_t)(mh * 8 * kWSBO), wo = (uint32_t)(n0 / 8) * sbo_w;
    const uint64_t dah = umma::make_desc(umma::smem_u32(a_hi) + ao, kLBO, kWSBO), dal = umma::make_desc(umma::smem_u32(a_lo) + ao, kLBO, kWSBO);
    const uint64_t dwh = umma::make_desc(umma::smem_u32(w_hi) + wo, kLBO, sbo_w), dwl = umma::make_desc(umma::smem_u32(w_lo) + wo, kLBO, sbo_w);
    umma::wg_gemm<0, 0>(tmem_d + (uint32_t)n0 + ((uint32_t)(64 * mh) << 16), false, dah, dal, dwh, dwl, (2 * kLBO) >> 4, (2 * kLBO) >> 4,
                        (8 * sbo_w) >> 4, Kp / 16, nn, false);
}

// Rows [m0, m0 + 64) x columns [c0, c0 + N) of this tile's dW_l in the issuing warpgroup's registers, then added in fixed point to the
// CTA's sums `dw` ([128 rows][LD columns] of the layer; `first`: the CTA's first tile, which sets them). Every slot belongs to one
// thread for the whole launch (the fragment position), so the read-modify-write needs no atomics. Each tile's product is rounded to
// the fixed-point grid before it is added, as a per-tile flush would round it: the totals do not depend on how tiles map to CTAs.
template <int N, int LD>
__device__ __forceinline__ void dw_rows_fx(unsigned long long* dw, int m0, int c0, uint64_t dzh, uint64_t dzl, uint64_t dah, uint64_t dal,
                                           bool first) {
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; i++) d[i] = 0.f;
    umma::wgmma_fence();
    // 16 samples = 2 eight-row groups per K step
    umma::wg_mma_regs<N, 1, 1>(d, dzh, dzl, dah, dal, (2 * kWSBO) >> 4, (2 * kWSBO) >> 4, kTile / 16, false);
    umma::wgmma_commit();
    umma::wgmma_wait0();
#pragma unroll
    for (int h = 0; h < 2; h++) {
        unsigned long long* p = dw + (size_t)frag_row(0, h) * LD + m0 * LD + c0;
#pragma unroll
        for (int j = 0; j < N / 8; j++) {
            ulonglong2* q = reinterpret_cast<ulonglong2*>(p + frag_col(j));
            ulonglong2 v = first ? make_ulonglong2(0ull, 0ull) : *q;
            v.x += fx_of(d[4 * j + 2 * h]);
            v.y += fx_of(d[4 * j + 2 * h + 1]);
            *q = v;
        }
    }
}
// dW_l = zbar^(l)^T a_l over the 128 samples of the tile: both tiles consumed as MN-major operands (one warpgroup, `half` = 0 / 1).
// M = 128: the two warpgroups take rows 0..63 / 64..127; M = 64: columns [0, na) / [na, N) of one M = 64 product. Added to the CTA's
// fixed-point sums (dw_rows_fx, row stride LD) in pieces of at most 32 columns (register budget); pieces `part`, part + parts, ... of
// the half (parts warpgroups share it).
template <int LD = 128>
__device__ __forceinline__ void issue_dw_w(unsigned long long* dw, int half, const uint8_t* z_hi, const uint8_t* a_hi, int M, int N, bool first,
                                           int part = 0, int parts = 1) {
    int m0 = 0, n0 = 0, nn = N;
    if (M == 128) m0 = 64 * half;
    else split_n(N, half, n0, nn);
    if (nn <= 0) return;
    const uint32_t zh = umma::smem_u32(z_hi) + (uint32_t)(m0 / 8) * kLBO;
    const uint64_t dzh = umma::make_desc(zh, kWSBO, kLBO), dzl = umma::make_desc(zh + kWTileBytes, kWSBO, kLBO);
    for (int p0 = 32 * part; p0 < nn; p0 += 32 * parts) {
        const uint32_t ah = umma::smem_u32(a_hi) + (uint32_t)((n0 + p0) / 8) * kLBO;
        const uint64_t dah = umma::make_desc(ah, kWSBO, kLBO), dal = umma::make_desc(ah + kWTileBytes, kWSBO, kLBO);
        if (nn - p0 >= 32) dw_rows_fx<32, LD>(dw, m0, n0 + p0, dzh, dzl, dah, dal, first);
        else dw_rows_fx<16, LD>(dw, m0, n0 + p0, dzh, dzl, dah, dal, first);
    }
}

// The CTA's sums of the slots issue_dw_w (same arguments) reads and writes in this thread -> L2, ahead of the products
__device__ __forceinline__ void prefetch_dw_w(const unsigned long long* dw, int half, int M, int N, int part, int parts) {
    int m0 = 0, n0 = 0, nn = N;
    if (M == 128) m0 = 64 * half;
    else split_n(N, half, n0, nn);
    for (int p0 = 32 * part; p0 < nn; p0 += 32 * parts)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (p0 + 8 * j < nn)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(dw + (size_t)(m0 + frag_row(0, h)) * 128 + n0 + p0 + frag_col(j)));
}

// Layer-0 operand tile of one sample row. Thread (row, grp) builds the 8-column cores grp, grp+4, ... of the lattice part and
// the two tail cores T_grp, T_{grp+4} (tail = concat points | SH | normal | geom, 64 columns = 8 cores after column 2L).
__device__ __forceinline__ void build_input_tile(const RgbParams& P, const LevelC* lc, const float2* __restrict__ lattice,
                                                 const float* __restrict__ pos, const float* __restrict__ dirs,
                                                 const float* __restrict__ sdf_grad, const float* __restrict__ geom, int n, bool valid, int row,
                                                 int grp, uint8_t* a_hi, uint8_t* a_lo) {
    float x[3] = {0.f, 0.f, 0.f};
    if (valid) { x[0] = pos[(size_t)n * 3]; x[1] = pos[(size_t)n * 3 + 1]; x[2] = pos[(size_t)n * 3 + 2]; }
    const int level_cores = P.L / 4;
    for (int kc = grp; kc < level_cores; kc += kRgbGroups) {
        float fv[8];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            Simplex3 s;
            float2 v[4];
            const float2 a = level_features(x, lc, kc * 4 + q, lattice, P.T, P.cap_mask, s, v);
            fv[2 * q] = a.x; fv[2 * q + 1] = a.y;
        }
        store8w(a_hi, a_lo, row, kc, fv);
    }
    // ---- tail cores
    float t0[8], t1[8];
    const float* gp = geom + (size_t)n * kGeomDim + grp * 8;
#pragma unroll
    for (int i = 0; i < 8; i++) t1[i] = valid ? gp[i] : 0.f;                 // T_{grp+4}: geom[8 grp .. 8 grp + 7]
    float sh[kShCols];
    {
        float dx = 0.f, dy = 0.f, dz = 0.f;
        if (valid) { dx = dirs[(size_t)n * 3]; dy = dirs[(size_t)n * 3 + 1]; dz = dirs[(size_t)n * 3 + 2]; }
        psdf::sh_eval(dx, dy, dz, 5, sh);
        if (!valid) {
#pragma unroll
            for (int i = 0; i < kShCols; i++) sh[i] = 0.f;
        }
    }
    if (grp == 0) {
        t0[0] = x[0] * P.points_scaling; t0[1] = x[1] * P.points_scaling; t0[2] = x[2] * P.points_scaling; t0[3] = 0.f;
        t0[4] = sh[0]; t0[5] = sh[1]; t0[6] = sh[2]; t0[7] = sh[3];
    } else if (grp == 1) {
#pragma unroll
        for (int i = 0; i < 8; i++) t0[i] = sh[4 + i];
    } else if (grp == 2) {
#pragma unroll
        for (int i = 0; i < 8; i++) t0[i] = sh[12 + i];
    } else {
#pragma unroll
        for (int i = 0; i < 5; i++) t0[i] = sh[20 + i];
        float gx = 0.f, gy = 0.f, gz = 0.f;
        if (valid) { gx = sdf_grad[(size_t)n * 3]; gy = sdf_grad[(size_t)n * 3 + 1]; gz = sdf_grad[(size_t)n * 3 + 2]; }
        const float inv = 1.0f / fmaxf(sqrtf(gx * gx + gy * gy + gz * gz), 1e-12f);       // F.normalize(eps = 1e-12)
        t0[5] = gx * inv; t0[6] = gy * inv; t0[7] = gz * inv;
    }
    store8w(a_hi, a_lo, row, level_cores + grp, t0);
    store8w(a_hi, a_lo, row, level_cores + 4 + grp, t1);
    // zero padding up to Kp[0] (in_dim is a multiple of 8; a multiple of 16 only for even L/4... pad the odd core)
    const int cores = P.g.Kp[0] / 8;
    for (int kc = level_cores + 8 + grp; kc < cores; kc += kRgbGroups) {
        float z8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        store8w(a_hi, a_lo, row, kc, z8);
    }
}

// Encoder backward of the colour-network-shaped backwards (no tangent term): lattice[l][idx_r] += window_l B_r abar_0[l] from the
// exchange rows their persistent kernels write, xch[l][tile * 128 + row] = abar_0's two columns of level l. blockIdx.y = level (blocks
// of one level run together: its gradient table stays in L2 while they land), warp = 32 consecutive sample slots, i.e. the rows of one
// warp of the per-row layout, so the match_any groups and the float peer sums are those of a scatter inside the persistent kernel. It runs
// with every warp slot of the SM occupied, where the persistent kernel's 16 warps per SM would wait on its dependent chains of simplex
// recompute, match_any, shuffle sums and reductions with the tensor cores idle. pos, scale and shift have D columns; fx_lattice:
// deterministic mode's fixed-point accumulators, else NULL.
constexpr int kScatterThreads = 256;
template <int D>
static __global__ void __launch_bounds__(kScatterThreads, 8)
k_lattice_scatter(int N, int T, unsigned cap_mask, const float* __restrict__ pos, const float2* __restrict__ xch, int xch_stride,
                  const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ window,
                  float* __restrict__ grad_lattice, unsigned long long* __restrict__ fx_lattice) {
    const int slot = blockIdx.x * kScatterThreads + threadIdx.x;
    if (slot >= xch_stride) return;                                  // whole warps (xch_stride % 128 == 0)
    const int l = blockIdx.y, lane = threadIdx.x & 31;
    const bool valid = slot < N;
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
    scatter_level<false, D>(x, nullptr, sc, sh, w, a.x, a.y, 0.f, 0.f, valid, aggregate, true, lane, cap_mask, (unsigned)T,
                            grad_lattice + (size_t)l * T * 2, fx_lattice ? fx_lattice + (size_t)l * T * 2 : nullptr);
}

}  // namespace psdf_rgb
