// Training backward of the fused colour network (sm_90a, wgmma): d loss / d (linear rgb) per sample in ->
// lattice gradient, d loss / d sdf-gradient (through the normalisation), d loss / d geom feature, weight + bias gradients of the 4
// linear layers. Replaces loss.backward() through RGB.forward (permuto_sdf_py/models/models.py:395-414) -- encoding backward,
// 4 x (GELU backward, 2 GEMMs), normalize / cat backward. Four kernels: the input-tile kernel k_rgb_input_tiles (48 warps per SM), the
// persistent tensor-core kernel below, the cross-CTA sum of its weight-gradient sums (k_dw_reduce, fused_common.cuh) and the
// full-occupancy lattice scatter k_lattice_scatter (fused_rgb_common.cuh, shared with the background backward).
//
// Per 128-sample tile (512 threads). Every product lands in the registers of the warpgroup that issues it: warpgroup (mh, nh) =
// (wgi & 1, wgi >> 1) forms rows 64 mh .. 64 mh + 63 x column half nh (split_n) and consumes them in place.
//   1. input tile a_0 (encoder gather + SH + normal + geom, built by k_rgb_input_tiles into the workspace) -> s_a by ONE TMA load
//      (64 KB / tile, loaded again for dW_0). The next tile's load is issued as soon as the step-0 products have read s_a;
//   2. forward recompute, layers 0..2: a_{l+1} = gelu(z^(l) + b_l) -> s_a straight from the fragments; the raw z^(l) go to this thread's
//      slots of the CTA's stash (global, L2 resident) and come back to the same thread in the reverse sweep: the reverse step l splits
//      its Kp_l = Np_{l-1} columns exactly as the forward layer l-1 split them, so it needs no barrier;
//   3. seed zbar^(3) = d loss / d linear rgb -> s_z;
//   4. reverse sweep l = 3..0, s_z = zbar^(l), s_a = a_l: abar_l = zbar^(l) W_l (transposed weight block as the B operand) and a share
//      of the WEIGHT GRADIENT dW_l = zbar^(l)^T a_l, formed on the tensor cores from the two tiles as they sit in shared memory (the
//      sample axis is the MMA K dimension and an operand tile in the K-major core-matrix layout is an MN-major operand for that
//      product, see fused_sdf_bwd.cu). Each warpgroup adds its dW pieces from its registers to the CTA's fixed-point sums (each slot
//      owned by one thread: no atomics); k_dw_reduce adds up the CTAs' sums after the launch -- with the same totals as a per-tile
//      fixed-point flush. After a barrier the fragments become zbar^(l-1) = abar_l gelu'(z^(l-1)) -> s_z, the bias gradient
//      (frag_pair_colsum: the bits of the per-row colsum16), and a_{l-1} is rebuilt into s_a from the stashed z^(l-2) (l = 3, 2) or
//      comes back by TMA (l = 1);
//   5. l = 0: abar_0's lattice columns leave from the registers to the exchange rows of the workspace ([level][tile * 128 + row]
//      float2, a thread's column pair is one level) for k_lattice_scatter; the normal and geom columns pass through a small fp32
//      staging tile over s_z to the per-row tail: normal -> sdf-gradient (= or +=), geom gradient.
// Deterministic mode (common.cuh): every gradient is summed in fixed point instead and added to the float gradients by the flush that
// follows the launches.
// Weights stream per layer through one 64 KB buffer by TMA; the next block is requested as soon as the MMAs that read the
// current one have retired, so the copy hides behind the epilogue.
// Stash of a CTA (float4 slots, slot index * 512 + tid): z^(l) fragments of layer l at [8 l, 8 l + 8). Weight-gradient sums: g_dw_rgb_bwd.
#include <cstdio>
#include <cstdlib>
#include "fused_common.cuh"
#include "fused_rgb_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;
using namespace psdf_rgb;

namespace {
constexpr int kStashSlots = 24;
__device__ float4 g_stash_rgb_bwd[(size_t)kAccCtas * kStashSlots * kRgbThreads];     // per-CTA stashes, 192 KB each
// weight-gradient sums of each CTA in fixed point (common.cuh fx_of), [CTA][layer][128 rows][128 columns]
constexpr int kDwSlots = kNL * 128 * 128;
__device__ unsigned long long g_dw_rgb_bwd[(size_t)kAccCtas * kDwSlots];
struct RgbDwSlab { static __device__ const void* get() { return g_dw_rgb_bwd; } };
constexpr int kFxW = kDetRgbW, kFxB = 4 * kDetRgbW;    // weight / bias offsets in DetBufs::rgb_mlp
constexpr int kRgbSpillBytes = 2 * kWTileBytes;      // [hi | lo] of one operand tile
constexpr int kTailCols = 3 + kGeomDim;              // abar_0 columns of the normal and the geom feature
constexpr int kTailLd = kTailCols + 1;               // row stride of their fp32 staging tile
constexpr int kBxBytes = 8 * 16 * 32 * sizeof(float);   // odd warps' fragments of the bias column sums, [8 warp pairs][16][32 lanes]

struct RgbSpill {
    const uint8_t* a0;   // [ntiles][64 KB] input tiles a_0 (k_rgb_input_tiles)
    float2* xch;         // [L][xch_stride] abar_0 of every level and sample slot (tile * 128 + row)
    int xch_stride;      // sample slots = ntiles * 128
    float* gbias[kNL];   // (+=)
    unsigned long long* fx_mlp;         // deterministic mode: fixed-point accumulators (DetBufs::rgb_mlp), else NULL
    unsigned long long* phase_cycles;   // [16] += clock64 deltas of thread 0 per phase (PSDF_PHASE_TIMING=1, diagnostics), else NULL
};
// phase ids of the diagnostic counters
enum { kPhTileLoad = 0, kPhForward0 = 1, kPhSeed = 4, kPhReverse3 = 5, kPhTail = 9, kPhFlush = 10, kPhTiles = 11 };
#define PSDF_PHASE(id)                                                                     \
    do {                                                                                   \
        if (sp.phase_cycles && tid == 0) {                                                 \
            const long long now_ = clock64();                                              \
            atomicAdd(sp.phase_cycles + (id), (unsigned long long)(now_ - phase_t0));      \
            phase_t0 = now_;                                                               \
        }                                                                                  \
    } while (0)

// rows 64 mh .. 64 mh + 63 x columns [n0, n0 + nn) of [128 x K] x [Nw x K]^T into the issuing warpgroup's registers: streams_product on
// the 128-column tiles (A = 128 rows with the 2048-byte row-group stride, weight block [Nw rows][K] K-major)
__device__ __forceinline__ void tile_product(float* acc, int nn, int mh, const uint8_t* a, const uint8_t* w_hi, const uint8_t* w_lo, int K, int n0) {
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = 0.f;
    const uint32_t ro = (uint32_t)(mh * 8 * kWSBO);
    switch (nn / 16) {
        case 1: streams_product<16, 1>(acc, a, 0, kWTileBytes, ro, w_hi, w_lo, K, n0, kWSBO); break;
        case 2: streams_product<32, 1>(acc, a, 0, kWTileBytes, ro, w_hi, w_lo, K, n0, kWSBO); break;
        case 3: streams_product<48, 1>(acc, a, 0, kWTileBytes, ro, w_hi, w_lo, K, n0, kWSBO); break;
        case 4: streams_product<64, 1>(acc, a, 0, kWTileBytes, ro, w_hi, w_lo, K, n0, kWSBO); break;
        default: break;
    }
}

// Layer-0 input tiles of every tile of the launch -> a0 ([tile][64 KB], the bytes build_input_tile writes into s_a in the forward):
// block = (tile, group) with one thread per row, so a warp is 32 consecutive rows of one group, as in the per-row layout of the persistent
// kernels. Cores past Kp[0] are not written.
constexpr int kInputTileThreads = kTile;
__global__ void __launch_bounds__(kInputTileThreads)
k_rgb_input_tiles(RgbParams P, const float* __restrict__ pos, const float* __restrict__ dirs, const float* __restrict__ sdf_grad,
                  const float* __restrict__ geom, const float2* __restrict__ lattice, const float* __restrict__ scale,
                  const float* __restrict__ shift, const float* __restrict__ window, uint8_t* __restrict__ a0) {
    __shared__ LevelC lc;
    load_level_consts(&lc, P.L, scale, shift, window, threadIdx.x, kInputTileThreads);
    __syncthreads();
    const int tile = blockIdx.x / kRgbGroups, grp = blockIdx.x % kRgbGroups, row = threadIdx.x;
    const int n = tile * kTile + row;
    uint8_t* t = a0 + (size_t)tile * kRgbSpillBytes;
    build_input_tile(P, &lc, lattice, pos, dirs, sdf_grad, geom, n, n < P.N, row, grp, t, t + kWTileBytes);
}

__global__ void __launch_bounds__(kRgbThreads, 1)
k_rgb_fused_backward(RgbParams P, const float* __restrict__ sdf_grad, const uint8_t* __restrict__ blob, const float* __restrict__ g_out,
                     float* __restrict__ g_sdf_grad, float* __restrict__ g_geom, RgbSpill sp) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_a = smem;                                   // activation tiles [hi | lo]
    uint8_t* s_z = s_a + 2 * kWTileBytes;                  // adjoint tiles [hi | lo]
    uint8_t* s_w = s_z + 2 * kWTileBytes;                  // weights of the current GEMM [hi | lo]
    float* s_bias = reinterpret_cast<float*>(s_w + 2 * kWTileBytes);      // 4 x 128
    // 4 x 128 bias-gradient accumulators of this CTA: float (s_gbf), or fixed point (s_gb) in deterministic mode
    unsigned long long* s_gb = reinterpret_cast<unsigned long long*>(s_bias + kNL * 128);
    float* s_gbf = reinterpret_cast<float*>(s_gb);
    const bool det = sp.fx_mlp != nullptr;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gb + kNL * 128);   // [0] weights, [1] a_0 reload for dW_0, [2] tile loads
    float* s_bx = reinterpret_cast<float*>(bars + 8);      // bias column sums: the odd warps' fragments (frag_pair_colsum)
    // staging tile of abar_0's normal | geom columns, [128][kTailLd] fp32 over s_z: written after the last reverse step's products,
    // the last readers of s_z in the tile, have completed
    float* s_tail = reinterpret_cast<float*>(s_z);

    const int tid = threadIdx.x, warp = warp_uniform(tid >> 5), lane = tid & 31;
    const int row = tid & 127, grp = tid >> 7;
    const int wgi = warp >> 2, mh = wgi & 1, nh = wgi >> 1;
    const int pair = 2 * wgi + ((warp & 3) >> 1);          // 32-row group of this warp's fragment rows
    float4* stash = g_stash_rgb_bwd + (size_t)blockIdx.x * kStashSlots * kRgbThreads + tid;     // this thread's slot 0
    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_init(&bars[1], 1);
        umma::mbar_init(&bars[2], 1);
        umma::mbar_fence_init();
    }
    for (int i = tid; i < kNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        s_bias[i] = (c < P.g.Np[l]) ? reinterpret_cast<const float*>(blob + P.g.bias[l])[c] : 0.0f;
        s_gb[i] = 0ull;        // also clears s_gbf
    }
    __syncthreads();
    uint32_t w_phase = 0, a0_phase = 0, tl_phase = 0;
    unsigned long long* dw_cta = g_dw_rgb_bwd + (size_t)blockIdx.x * kDwSlots;    // this CTA's weight-gradient sums, layer l at l * 128 * 128

    const int ntiles = (P.N + kTile - 1) / kTile;
    if (tid == 0 && blockIdx.x < ntiles) {
        load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
        umma::mbar_expect_tx(&bars[2], (uint32_t)kRgbSpillBytes);
        umma::bulk_g2s(s_a, sp.a0 + (size_t)blockIdx.x * kRgbSpillBytes, (uint32_t)kRgbSpillBytes, &bars[2]);
    }
    long long phase_t0 = sp.phase_cycles ? clock64() : 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const bool first_tile = tile == (int)blockIdx.x;
        const int n = tile * kTile + row;
        const bool valid = n < P.N;
        // a_0 of this tile -> s_a (TMA load issued next to the first weight load or after the previous tile's step 0)
        umma::mbar_wait(&bars[2], tl_phase);
        tl_phase ^= 1;
        PSDF_PHASE(kPhTileLoad);

        // ---------------- forward recompute, layers 0..2
#pragma unroll 1
        for (int l = 0; l < 3; l++) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            const int Np = warp_uniform(P.g.Np[l]), Kp = warp_uniform(P.g.Kp[l]);
            int n0, nn;
            split_n(Np, nh, n0, nn);
            float acc[32];
            tile_product(acc, nn, mh, s_a, s_w, s_w + Np * Kp * 2, Kp, n0);
            __syncthreads();                                       // every product has read s_a and s_w
            if (tid == 0) load_layer_weights(s_w, blob, P.g, l < 2 ? l + 1 : 3, l == 2, &bars[0]);   // W_{l+1}, then W_3^T
            // raw z^(l) -> this thread's stash slots (read back by this thread in the reverse steps l + 1 and l + 2), a_{l+1} -> s_a
#pragma unroll
            for (int j = 0; j < 8; j++)
                if (8 * j < nn) stash[(8 * l + j) * kRgbThreads] = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                if (8 * j < nn) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int r = frag_row(mh, h), c = n0 + frag_col(j);
                        float a[2];
#pragma unroll
                        for (int b = 0; b < 2; b++) {
                            const float zz = acc[4 * j + 2 * h + b] + s_bias[l * 128 + c + b];
                            a[b] = zz * gelu_eval(zz).cdf;
                        }
                        store_pair(s_a, s_a + kWTileBytes, r, c, a[0], a[1], kWSBO);
                    }
                }
            }
            PSDF_PHASE(kPhForward0 + l);
        }
        // ---------------- seed: zbar^(3) = d loss / d linear rgb (3 of 16 padded columns)
        if (grp == 0) {
            float zb[16];
#pragma unroll
            for (int i = 0; i < 16; i++) zb[i] = (i < 3 && valid) ? g_out[(size_t)n * 3 + i] : 0.f;
            store8w(s_z, s_z + kWTileBytes, row, 0, zb);
            store8w(s_z, s_z + kWTileBytes, row, 1, zb + 8);
            int col;
            const float cs = colsum16(zb, lane, col);
            if (!(lane & 1) && col < 3) {
                if (det) fx_add(&s_gb[3 * 128 + col], cs);
                else atomicAdd(&s_gbf[3 * 128 + col], cs);
            }
        }
        PSDF_PHASE(kPhSeed);
        // ---------------- reverse sweep, layers 3..0: s_z = zbar^(l), s_a = a_l
        const bool rvalid0 = tile * kTile + frag_row(mh, 0) < P.N, rvalid1 = tile * kTile + frag_row(mh, 1) < P.N;   // fragment rows
#pragma unroll 1
        for (int l = 3; l >= 0; l--) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            if (l == 0) umma::mbar_wait(&bars[1], a0_phase);      // a_0 is back in s_a
            umma::fence_async_smem();
            __syncthreads();
            const int Np = warp_uniform(P.g.Np[l]), Kp = warp_uniform(P.g.Kp[l]);
            if (!first_tile) prefetch_dw_w(dw_cta + l * 128 * 128, mh, Np > 64 ? 128 : 64, Kp, nh, 2);
            int n0, nn;
            split_n(Kp, nh, n0, nn);
            float acc[32];
            // abar_l [128 x Kp] = zbar^(l) [128 x Np] W_l: B operand = W_l^T stored [Kp rows][Np]
            tile_product(acc, nn, mh, s_z, s_w, s_w + Np * Kp * 2, Np, n0);
            // dW_l: the row half mh, every other 32-column piece of it
            issue_dw_w(dw_cta + l * 128 * 128, mh, s_z, s_a, Np > 64 ? 128 : 64, Kp, first_tile, nh, 2);
            __syncthreads();                                       // every product of this step has read s_z, s_a and s_w
            if (tid == 0) {
                if (l > 0) load_layer_weights(s_w, blob, P.g, l - 1, true, &bars[0]);
                else if (tile + (int)gridDim.x < ntiles) {       // the next tile's W_0 and, s_a being free, its a_0
                    load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
                    umma::mbar_expect_tx(&bars[2], (uint32_t)kRgbSpillBytes);
                    umma::bulk_g2s(s_a, sp.a0 + (size_t)(tile + gridDim.x) * kRgbSpillBytes, (uint32_t)kRgbSpillBytes, &bars[2]);
                }
                if (l == 1) {                  // s_a is free: a_0 returns by TMA for the last step
                    umma::mbar_expect_tx(&bars[1], (uint32_t)kRgbSpillBytes);
                    umma::bulk_g2s(s_a, sp.a0 + (size_t)tile * kRgbSpillBytes, (uint32_t)kRgbSpillBytes, &bars[1]);
                }
            }
            if (l > 0) {
                // zbar^(l-1) = abar_l gelu'(z^(l-1)) -> s_z from this thread's stashed z^(l-1); acc keeps it on the valid rows (0 elsewhere)
                // for the bias gradient of layer l - 1
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    if (8 * j < nn) {
                        const float4 z4 = stash[(8 * (l - 1) + j) * kRgbThreads];
                        const float z[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int r = frag_row(mh, h), c = n0 + frag_col(j);
                            float zb[2];
#pragma unroll
                            for (int b = 0; b < 2; b++) {
                                const int i = 4 * j + 2 * h + b;
                                const float zz = z[2 * h + b] + s_bias[(l - 1) * 128 + c + b];
                                const GeluEval ge = gelu_eval(zz);
                                zb[b] = acc[i] * fmaf(zz, ge.pdf, ge.cdf);
                                acc[i] = (h ? rvalid1 : rvalid0) ? zb[b] : 0.f;
                            }
                            store_pair(s_z, s_z + kWTileBytes, r, c, zb[0], zb[1], kWSBO);
                        }
                    }
                }
                // bias gradient of layer l - 1: column sums over each 32-row group, 32 columns at a time
#pragma unroll
                for (int q = 0; q < 2; q++) {
                    if (32 * q < nn) {
                        if (q) umma::bar_sync(1 + pair, 64);       // the even warp has read the first block's exchange
                        float cs;
                        int col;
                        if (frag_pair_colsum(acc + 16 * q, nn - 32 * q, s_bx + pair * 16 * 32, 1 + pair, cs, col)) {
                            if (det) fx_add(&s_gb[(l - 1) * 128 + n0 + 32 * q + col], cs);
                            else atomicAdd(&s_gbf[(l - 1) * 128 + n0 + 32 * q + col], cs);
                        }
                    }
                }
                if (l >= 2) {
                    // a_{l-1} = gelu(z^(l-2)) -> s_a from this thread's stashed z^(l-2) (the forward layer l - 2 split its columns as the
                    // reverse step l - 1 does)
                    int m0, mn;
                    split_n(P.g.Np[l - 2], nh, m0, mn);
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (8 * j < mn) {
                            const float4 z4 = stash[(8 * (l - 2) + j) * kRgbThreads];
                            const float z[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const int r = frag_row(mh, h), c = m0 + frag_col(j);
                                float a[2];
#pragma unroll
                                for (int b = 0; b < 2; b++) {
                                    const float zz = z[2 * h + b] + s_bias[(l - 2) * 128 + c + b];
                                    a[b] = zz * gelu_eval(zz).cdf;
                                }
                                store_pair(s_a, s_a + kWTileBytes, r, c, a[0], a[1], kWSBO);
                            }
                        }
                    }
                }
            } else {
                // abar_0: lattice columns -> the exchange rows (a thread's column pair is one level), normal | geom -> the staging tile
                const int tail0 = P.enc_cols + kShCols;
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    if (8 * j < nn) {
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int r = frag_row(mh, h), c = n0 + frag_col(j), i = 4 * j + 2 * h;
                            if (c < 2 * P.L) sp.xch[(size_t)(c >> 1) * sp.xch_stride + tile * kTile + r] = make_float2(acc[i], acc[i + 1]);
#pragma unroll
                            for (int b = 0; b < 2; b++)
                                if (c + b >= tail0 && c + b < tail0 + kTailCols) s_tail[r * kTailLd + c + b - tail0] = acc[i + b];
                        }
                    }
                }
            }
            PSDF_PHASE(kPhReverse3 + (3 - l));
        }
        a0_phase ^= 1;
        __syncthreads();
        // ---------------- tail: normal -> sdf-gradient, geom gradient (per row)
        if (valid) {
            const float* xr = s_tail + row * kTailLd;
            if (g_geom) {
                float* gg = g_geom + (size_t)n * kGeomDim + grp * 8;
#pragma unroll
                for (int i = 0; i < 8; i++) gg[i] = xr[3 + grp * 8 + i];
            }
            if (grp == 3 && g_sdf_grad) {
                const float gx = sdf_grad[(size_t)n * 3], gy = sdf_grad[(size_t)n * 3 + 1], gz = sdf_grad[(size_t)n * 3 + 2];
                const float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
                const float inv = 1.0f / fmaxf(nrm, 1e-12f);
                const float bx = xr[0], by = xr[1], bz = xr[2];
                float ox = bx * inv, oy = by * inv, oz = bz * inv;
                if (nrm > 1e-12f) {           // d (g / |g|) : (I - n n^T) / |g|
                    const float nx = gx * inv, ny = gy * inv, nz = gz * inv;
                    const float d = nx * bx + ny * by + nz * bz;
                    ox -= nx * d * inv; oy -= ny * d * inv; oz -= nz * d * inv;
                }
                float* o = g_sdf_grad + (size_t)n * 3;
                if (P.acc_sdf_grad) { o[0] += ox; o[1] += oy; o[2] += oz; }
                else { o[0] = ox; o[1] = oy; o[2] = oz; }
            }
        }
        // no barrier before the next tile: s_a was last read by this tile's step-0 products (the next tile's a_0 arrives by TMA, behind
        // the mbarrier), s_tail (over s_z) is next written by the next tile's seed, several barriers later
        PSDF_PHASE(kPhTail);
        if (sp.phase_cycles && tid == 0) atomicAdd(sp.phase_cycles + kPhTiles, 1ull);
    }
    __syncthreads();
    // ---- bias gradients of this CTA (the weight-gradient sums are added up across CTAs by k_dw_reduce)
    for (int i = tid; i < kNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        if (det) { if (c < P.g.N[l] && s_gb[i] != 0ull) atomicAdd(sp.fx_mlp + kFxB + l * 128 + c, s_gb[i]); }
        else if (c < P.g.N[l] && s_gbf[i] != 0.0f) atomicAdd(sp.gbias[l] + c, s_gbf[i]);
    }
    PSDF_PHASE(kPhFlush);
}

#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {

// workspace per 128-sample tile: the input operand tile a_0 (64 KB), written by k_rgb_input_tiles and loaded by TMA into the persistent
// kernel twice (forward recompute and the first layer's weight gradient), and the exchange rows of abar_0 (8 bytes per sample and level, sized for kMaxLevels
// so that the size depends on the sample count alone)
long long psdf_rgb_fused_backward_workspace_bytes(int N) {
    const int ntiles = div_up(N > 0 ? N : 1, kTile);
    return (long long)ntiles * (kRgbSpillBytes + (long long)kTile * kMaxLevels * sizeof(float2));
}

static int rgb_backward_impl(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                            const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                            int h1, int h2, int h3, const uint8_t* blob, const float* g_out, float* grad_lattice, float* g_sdf_grad,
                            float* g_geom, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1,
                            float* gb2, float* gb3, int accumulate_sdf_grad, void* stream) {
    RgbParams P;
    int rc = make_rgb_params(P, N, L, T, geom_dim, points_scaling, h1, h2, h3);
    if (rc != PSDF_OK) return rc;
    P.acc_sdf_grad = accumulate_sdf_grad ? 1 : 0;
    if (N == 0) return PSDF_OK;
    static_assert((size_t)kTile * kTailLd * 4 <= (size_t)2 * kWTileBytes, "the tail staging tile fits in s_z");
    const DetBufs* dbuf = det_buffers();
    if (dbuf && (long long)L * T * 2 > dbuf->lattice_len) return PSDF_ERR_UNSUPPORTED;   // reserve more with psdf_set_deterministic
    RgbSpill sp;
    float* b[kNL] = {gb0, gb1, gb2, gb3};
    float* w[kNL] = {gW0, gW1, gW2, gW3};
    for (int l = 0; l < kNL; l++) sp.gbias[l] = b[l];
    sp.fx_mlp = dbuf ? dbuf->rgb_mlp : nullptr;
    const int ntiles = div_up(N, kTile);
    uint8_t* a0 = workspace;
    sp.a0 = a0;
    sp.xch = reinterpret_cast<float2*>(workspace + (size_t)ntiles * kRgbSpillBytes);
    sp.xch_stride = ntiles * kTile;
    // diagnostics: PSDF_PHASE_TIMING=1 prints thread 0's clock64 breakdown per phase (average cycles per tile) after every launch
    static const bool timing = getenv("PSDF_PHASE_TIMING") && atoi(getenv("PSDF_PHASE_TIMING")) != 0;
    static unsigned long long* d_cycles = nullptr;
    static cudaEvent_t ev[5];
    sp.phase_cycles = nullptr;
    if (timing) {
        if (!d_cycles) {
            cudaMalloc(&d_cycles, 16 * sizeof(unsigned long long));
            for (auto& e : ev) cudaEventCreate(&e);
        }
        cudaMemsetAsync(d_cycles, 0, 16 * sizeof(unsigned long long), ST);
        sp.phase_cycles = d_cycles;
        cudaEventRecord(ev[0], ST);
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = (size_t)6 * kWTileBytes + kNL * 128 * (sizeof(float) + sizeof(unsigned long long)) + 64 + kBxBytes;
    // per device: set on every call (a second GPU needs its own opt-in)
    { static bool optin_[64]; psdf::psdf_optin_smem(k_rgb_fused_backward, 227 * 1024, optin_); }
    const int ctas = min(min(ntiles, sms), kAccCtas);
    k_rgb_input_tiles<<<ntiles * kRgbGroups, kInputTileThreads, 0, ST>>>(P, pos, dirs, sdf_grad, geom, reinterpret_cast<const float2*>(lattice),
                                                                         scale_factor, shift, window, a0);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[1], ST);
    k_rgb_fused_backward<<<ctas, kRgbThreads, smem, ST>>>(P, sdf_grad, blob, g_out, g_sdf_grad, g_geom, sp);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[2], ST);
    DwSums ds;
    for (int l = 0; l < kNL; l++) ds.gW[l] = w[l];
    ds.fx_mlp = sp.fx_mlp;
    ds.fx_w = kFxW;
    int max_nk = 0;
    for (int l = 0; l < kNL; l++) max_nk = max(max_nk, P.g.N[l] * P.g.K[l]);
    k_dw_reduce<128, unsigned long long, RgbDwSlab><<<dim3(div_up(max_nk, kDwReduceThreads), kNL, kDwReduceChunks), kDwReduceThreads, 0, ST>>>(
        P.g, ctas, ds);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[3], ST);
    k_lattice_scatter<3><<<dim3(div_up(sp.xch_stride, kScatterThreads), L), kScatterThreads, 0, ST>>>(
        N, T, P.cap_mask, pos, sp.xch, sp.xch_stride, scale_factor, shift, window, grad_lattice, dbuf ? dbuf->rgb_lattice : nullptr);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[4], ST);
    if (dbuf) {      // deterministic mode: fixed-point totals -> the float gradients (+=)
        FxSegs F;
        F.add(dbuf->rgb_lattice, grad_lattice, (long long)L * T * 2);
        for (int l = 0; l < kNL; l++) {
            F.add(dbuf->rgb_mlp + l * kFxW, w[l], (long long)P.g.N[l] * P.g.K[l]);
            F.add(dbuf->rgb_mlp + kFxB + l * 128, b[l], P.g.N[l]);
        }
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    if (timing) {
        unsigned long long h[16];
        cudaMemcpyAsync(h, d_cycles, sizeof(h), cudaMemcpyDeviceToHost, ST);
        cudaStreamSynchronize(ST);
        const double t = h[kPhTiles] ? (double)h[kPhTiles] : 1.0;
        float ms[4] = {0.f, 0.f, 0.f, 0.f};
        for (int i = 0; i < 4; i++) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
        fprintf(stderr, "[psdf_rgb_fused_backward N=%d tiles=%llu] cycles/tile: tile load wait %.0f forward %.0f %.0f %.0f seed %.0f rev3 %.0f rev2 %.0f rev1 %.0f "
                        "rev0 %.0f tail %.0f | flush/CTA %.0f | input tiles %.3f ms, fused kernel %.3f ms, weight-gradient reduction %.3f ms, "
                        "lattice scatter %.3f ms\n", N, h[kPhTiles], h[0] / t, h[1] / t, h[2] / t, h[3] / t, h[4] / t, h[5] / t, h[6] / t,
                h[7] / t, h[8] / t, h[9] / t, (double)h[kPhFlush] / ctas, ms[0], ms[1], ms[2], ms[3]);
    }
    return PSDF_OK;
}

int psdf_rgb_fused_backward(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                            const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                            int h1, int h2, int h3, const uint8_t* blob, const float* g_out, float* grad_lattice, float* g_sdf_grad,
                            float* g_geom, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1,
                            float* gb2, float* gb3, void* stream) {
    return rgb_backward_impl(N, L, T, pos, dirs, sdf_grad, geom, geom_dim, lattice, scale_factor, shift, window, points_scaling, h1, h2, h3, blob,
                             g_out, grad_lattice, g_sdf_grad, g_geom, workspace, gW0, gW1, gW2, gW3, gb0, gb1, gb2, gb3, 0, stream);
}
// same, with g_sdf_grad accumulated (+=): the buffer already holds d loss / d sdf_grad of the compositing and curvature terms
int psdf_rgb_fused_backward_acc(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                                const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                                int h1, int h2, int h3, const uint8_t* blob, const float* g_out, float* grad_lattice, float* g_sdf_grad,
                                float* g_geom, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1,
                                float* gb2, float* gb3, void* stream) {
    return rgb_backward_impl(N, L, T, pos, dirs, sdf_grad, geom, geom_dim, lattice, scale_factor, shift, window, points_scaling, h1, h2, h3, blob,
                             g_out, grad_lattice, g_sdf_grad, g_geom, workspace, gW0, gW1, gW2, gW3, gb0, gb1, gb2, gb3, 1, stream);
}

}  // extern "C"
