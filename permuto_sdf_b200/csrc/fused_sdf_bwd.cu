// Training backward of the fused encoding + SDF MLP (sm_90a, wgmma): given d loss / d {sdf, d sdf/dx, geom}
// per sample it produces the lattice gradient, the bias gradients and the weight gradients. Two kernels: the persistent
// tensor-core kernel forms the weight-gradient products from the operand tiles while they are still in shared memory
// (accumulated in the CTA's accumulator area, umma.cuh, over all tiles of the CTA) and hands abar_0 | tabar_0 to a
// full-occupancy kernel that scatters them into the lattice gradient.
//
// What it replaces in the reference: `loss.backward()` through SDF.get_sdf_and_gradient
// (permuto_sdf_py/models/models.py:199-259, create_graph=True) -- i.e. the double backward of the
// encoding (positions-gradient -> lattice) and of the 4-layer GELU MLP, ~60 PyTorch kernels per call.
//
// Math. The forward is y = MLP(enc(x)) (sdf = y0, geom = y1..), g = d sdf/dx. For fixed upstream gradients
// (ybar, gbar) the loss depends on the parameters through y and through the scalar s = gbar . g = D_v sdf, the
// directional derivative of sdf along v = gbar. So ONE tangent stream along v is enough (the forward kernel needs
// three because it must output g itself). With a_0 = enc(x), ta_0 = D_v enc(x) and for l = 0..3 (W_3 = output layer)
//     z_{l+1} = W_l a_l + b_l,  a_{l+1} = gelu(z_{l+1});     tz_{l+1} = W_l ta_l,  ta_{l+1} = gelu'(z_{l+1}) tz_{l+1},
// reverse mode gives (zbar_4 = ybar, tzbar_4 = e_0):
//     abar_l = W_l^T zbar_{l+1},   tabar_l = W_l^T tzbar_{l+1}
//     tzbar_l = gelu'(z_l) tabar_l
//     zbar_l  = gelu'(z_l) abar_l + gelu''(z_l) tz_l tabar_l
//     dW_l = zbar_{l+1} a_l^T + tzbar_{l+1} ta_l^T,   db_l = sum zbar_{l+1}
//     lattice[lvl][idx_r] += window_lvl (B_r abar_0[lvl] + dB_r tabar_0[lvl])       (B barycentric weights, dB their tangent)
//
// Per 128-sample tile (512 threads: row = tid & 127, group g = tid >> 7 owns operand cores g, g+4, .. in the encoder phases
// and the 16-column chunk g in the epilogues). Two 64 KB operand-tile buffers X, Y ([value hi | value lo | tangent hi | tangent lo]):
//   1. encoder: a_0, ta_0 -> X; X leaves by ONE TMA store (64 KB / tile, re-read from L2 in step 4: the only spill left)
//   2. forward recompute, layers 0..2: each warpgroup forms a row half x column half of both streams in its registers (value and tangent
//      of one (row, column) in the same thread) and writes a_1 -> Y, a_2 -> X, a_3 -> Y straight from the fragments; the raw z_1, z_2
//      (value + tangent) STAY in the accumulator area (4 x 64 columns), z_3 passes through the work columns to give gelu'(z_3),
//      gelu''(z_3) tz_3 in registers (layer 3 is reversed right away)
//   3. seed zbar_4 -> X
//   4. reverse sweep l = 3..0:  abar_l = zbar_{l+1} W_l uses the FORWARD weight tile as an MN-major B operand (no transposed
//      copy, weights resident for the CTA's lifetime); while it runs, a_l / ta_l are rebuilt into Y from the stored z_l
//      (l = 2, 1) or come back by TMA (l = 0); then dW_l += zbar_{l+1}^T a_l: the sample axis is the MMA K dimension and a
//      K-major operand tile IS an MN-major operand for that product, so X and Y are multiplied as they sit. The four dW
//      accumulators (M = 64) share 2 x 64 columns: an M = 64 product is stored to lanes (m / 16) * 32 + m % 16, so a second
//      accumulator lives at lane offset 16 of the same columns (tests/test_umma_probe_gpu.py).
//      In the last step (l = 0) abar_0 | tabar_0 leave from the registers to the exchange region of the workspace, one float4
//      (a0, a1, t0, t1) per level and sample, [level][sample slot]: a warp's 32 rows of one level are one contiguous 512-byte store.
// The encoder backward is its own launch, k_sdf_lattice_scatter: warp-aggregated red.global.add.v2.f32 into the lattice gradient.
// Inside the persistent kernel it was the longest phase of a tile (one CTA of 16 warps per SM, tensor cores idle, long dependent chains
// of simplex recompute, match_any, shuffle sums and reductions); on its own it runs with every warp slot of the SM occupied. Its warps
// are the rows of the persistent kernel's warps, so the match_any groups and the float peer sums are the same.
// Deterministic mode (common.cuh): every gradient (lattice, weights, biases) is summed in fixed point instead and added to the float
// gradients by the flush that follows the two launches.
// Accumulator map (512 columns): [0,256) z_1 | tz_1 | z_2 | tz_2, [256,384) work (value | tangent), [384,512) dW_0/dW_1, dW_2/dW_3.
#include <cstdio>
#include <cstdlib>
#include "fused_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;

namespace {
constexpr int kBwdThreads = 512;
constexpr int kGroups = kBwdThreads / kTile;
constexpr int kSetBytes = 4 * kATileBytes;         // one operand tile set [value hi | value lo | tangent hi | tangent lo]
constexpr uint32_t kColWork = 256, kColDw = 384;
__device__ float g_acc_bwd[(size_t)kAccCtas * kTile * 512];     // accumulator areas (umma.cuh)
constexpr int kFxW = kDetSdfW, kFxB = 4 * kDetSdfW;    // weight / bias offsets in DetBufs::sdf_mlp

struct BwdOut {
    uint8_t* a0_spill;  // [ntiles][64 KB] encoder operand tiles, written and re-read by the same CTA
    float4* xch;        // [L][xch_stride] abar_0 | tabar_0 (a0, a1, t0, t1) per level and sample slot (tile * 128 + row)
    int xch_stride;     // sample slots = ntiles * 128
    float* gW[kNL];     // [N_l, K_l] (+=)
    float* gbias[kNL];  // [N_l]      (+=)
    unsigned long long* fx_mlp;       // deterministic mode: fixed-point accumulators (DetBufs::sdf_mlp), else NULL
    unsigned long long* phase_cycles;   // [16] += clock64 deltas of thread 0 per phase (PSDF_PHASE_TIMING=1, diagnostics), else NULL
};
// Up to kMaxSeg independent sample sets (the main samples, the curvature pass' shifted samples, the off-surface points of one training
// iteration) are processed by ONE launch: every set starts on a tile boundary, so the sets share one last partial wave instead of
// one each.
constexpr int kMaxSeg = 3;
struct Segments {
    int n[kMaxSeg];          // samples of the set
    int tile0[kMaxSeg + 1];  // first tile of the set (prefix sum of ceil(n / 128))
    const float* pos[kMaxSeg];
    const float* g_sdf[kMaxSeg];
    const float* g_grad[kMaxSeg];
    const float* g_geom[kMaxSeg];
};
// phase ids of the diagnostic counters
enum { kPhEncoder = 0, kPhForward = 1, kPhSeed = 2, kPhReverse3 = 3, kPhReverse2 = 4, kPhReverse1 = 5, kPhReverse0 = 6, kPhFlush = 7,
       kPhTiles = 8 };
#define PSDF_PHASE(id)                                                                     \
    do {                                                                                   \
        if (out.phase_cycles && tid == 0) {                                                \
            const long long now_ = clock64();                                              \
            atomicAdd(out.phase_cycles + (id), (unsigned long long)(now_ - phase_t0));     \
            phase_t0 = now_;                                                               \
        }                                                                                  \
    } while (0)

// in place for 16 accumulator columns (zz = z + bias): z <- a = gelu(zz), tz <- ta = gelu'(zz) tz; g1 = gelu'(zz), g2t = gelu''(zz) tz
__device__ __forceinline__ void activations16(float* z, float* tz, const float* bias, float* g1, float* g2t) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const float zz = z[i] + bias[i];
        const GeluEval ge = gelu_eval(zz);
        const float d1 = fmaf(zz, ge.pdf, ge.cdf);
        g2t[i] = ge.pdf * (2.0f - zz * zz) * tz[i];
        z[i] = zz * ge.cdf;
        tz[i] = d1 * tz[i];
        g1[i] = d1;
    }
}
__device__ __forceinline__ void store_set16(uint8_t* set, int row, int c, const float* a, const float* ta) {
    store8(set, set + kATileBytes, row, 2 * c, a);
    store8(set, set + kATileBytes, row, 2 * c + 1, a + 8);
    store8(set + 2 * kATileBytes, set + 3 * kATileBytes, row, 2 * c, ta);
    store8(set + 2 * kATileBytes, set + 3 * kATileBytes, row, 2 * c + 1, ta + 8);
}

// The wgmma sequences of a reverse step are issued by several warpgroups: warpgroups 0 / 1 issue the value / tangent stream of the
// reverse GEMM, warpgroups 2 / 3 one half of the weight-gradient columns each. Every issuer owns its accumulator columns and
// all its threads arrive on the phase's mbarrier (initialised with the issuers' thread count) once the results are stored.
// one stream of  abar[128 x Kp] = zbar[128 x Np] W : A = zbar tiles K-major, B = the FORWARD weight tile [Np rows][Kp] read as an
// MN-major operand (reduction over the rows: 8-row groups are sbo_w apart, the k cores kLBO); both row halves, one warpgroup
__device__ __forceinline__ void issue_reverse(uint32_t tmem_d, const uint8_t* z_hi, const uint8_t* z_lo, const uint8_t* w_hi,
                                              const uint8_t* w_lo, int Kp, int Np) {
    const uint32_t sbo_w = (Kp / 8) * kLBO;
    const uint64_t dwh = umma::make_desc(umma::smem_u32(w_hi), sbo_w, kLBO), dwl = umma::make_desc(umma::smem_u32(w_lo), sbo_w, kLBO);
    for (int mh = 0; mh < 2; mh++) {
        const uint32_t ao = (uint32_t)(mh * 8 * kSBO_A);
        const uint64_t dzh = umma::make_desc(umma::smem_u32(z_hi) + ao, kLBO, kSBO_A), dzl = umma::make_desc(umma::smem_u32(z_lo) + ao, kLBO, kSBO_A);
        umma::wg_gemm<0, 1>(tmem_d + ((uint32_t)(64 * mh) << 16), false, dzh, dzl, dwh, dwl, (2 * kLBO) >> 4, (2 * sbo_w) >> 4, (8 * kLBO) >> 4,
                            Np / 16, Kp, false);
    }
}
// columns [n0, n0 + nn) of  dW (+)= zbar^T a + tzbar^T ta : both tile sets consumed as MN-major operands, K = the 128 samples, M = 64
// (one warpgroup)
__device__ __forceinline__ void issue_dw_part(uint32_t tmem_d, const uint8_t* zset, const uint8_t* aset, int n0, int nn, bool clear) {
    if (nn <= 0) return;
    const uint32_t aoff = (n0 / 8) * kLBO;
#pragma unroll 1
    for (int s = 0; s < 2; s++) {
        const uint64_t dzh = umma::make_desc(umma::smem_u32(zset + s * 2 * kATileBytes), kSBO_A, kLBO);
        const uint64_t dzl = umma::make_desc(umma::smem_u32(zset + s * 2 * kATileBytes + kATileBytes), kSBO_A, kLBO);
        const uint64_t dah = umma::make_desc(umma::smem_u32(aset + s * 2 * kATileBytes) + aoff, kSBO_A, kLBO);
        const uint64_t dal = umma::make_desc(umma::smem_u32(aset + s * 2 * kATileBytes + kATileBytes) + aoff, kSBO_A, kLBO);
        // 16 samples = two 8-sample groups per K step
        umma::wg_gemm<1, 1>(tmem_d + n0, true, dzh, dzl, dah, dal, (2 * kSBO_A) >> 4, (2 * kSBO_A) >> 4, (8 * kLBO) >> 4, kTile / 16, nn,
                            !(clear && s == 0));
    }
}

// D = 3: positions [N,3]; D = 4: space-time positions [N,4] with the tangent along (g_grad, 0) (g_grad holds spatial derivatives)
template <int D>
__global__ void __launch_bounds__(kBwdThreads, 1)
k_sdf_fused_backward(FusedParams P, Segments S, const float2* __restrict__ lattice, const float* __restrict__ scale,
                     const float* __restrict__ shift, const float* __restrict__ window, const uint8_t* __restrict__ blob, BwdOut out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_w = smem;                                   // forward operand blob (weights hi/lo + biases), resident
    uint8_t* s_X = smem + P.g.total;
    uint8_t* s_Y = s_X + kSetBytes;
    LevelC* lc = reinterpret_cast<LevelC*>(s_Y + kSetBytes);
    // 4 x 64 bias-gradient accumulators of this CTA: float (s_gbf), or fixed point (s_gb) in deterministic mode
    unsigned long long* s_gb = reinterpret_cast<unsigned long long*>(lc + 1);
    float* s_gbf = reinterpret_cast<float*>(s_gb);
    const bool det = out.fx_mlp != nullptr;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gb + kNL * 64);   // [0] TMA loads, [1] mma, [2] dW mma
    float* s_seed = reinterpret_cast<float*>(bars + 5);   // [128][(out_dim - 1) | 1] upstream d loss / d geom of the tile (coalesced copy)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row = tid & 127, grp = tid >> 7;
    const int level_cores = P.L / 4;
    const int K0 = P.g.Kp[0];
    const int wgi = warp >> 2;
    const bool gemm_issuer = wgi < 2;                      // stream = warpgroup
    const bool dw_issuer = wgi >= 2;                       // column half = warpgroup - 2

    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_init(&bars[1], 2 * 128);
        umma::mbar_init(&bars[2], 2 * 128);
        umma::mbar_fence_init();
        umma::acc_attach(g_acc_bwd + (size_t)blockIdx.x * kTile * 512, 512);
    }
    load_level_consts<D>(lc, P.L, scale, shift, window, tid, kBwdThreads);
    for (int i = tid; i < kNL * 64; i += kBwdThreads) s_gb[i] = 0ull;     // also clears s_gbf
    __syncthreads();
    if (tid == 0) {
        umma::mbar_expect_tx(&bars[0], (uint32_t)P.g.total);
        umma::bulk_g2s(s_w, blob, (uint32_t)P.g.total, &bars[0]);
    }
    __syncthreads();
    const uint32_t tmem_base = 0;
    const uint32_t tlane = tmem_base + ((uint32_t)((warp & 3) * 32) << 16);     // this warp's 32 accumulator lanes
    umma::mbar_wait(&bars[0], 0);
    uint32_t ld_phase = 1, mma_phase = 0, dw_phase = 0;

    const int ntiles = S.tile0[kMaxSeg];
    bool first_tile = true;
    long long phase_t0 = out.phase_cycles ? clock64() : 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, first_tile = false) {
        const int seg = tile >= S.tile0[2] ? 2 : (tile >= S.tile0[1] ? 1 : 0);
#define PSDF_SEG(f) (seg == 2 ? S.f[2] : (seg == 1 ? S.f[1] : S.f[0]))     // no dynamic indexing of the parameter struct (local-memory copy)
        const int seg_tile0 = PSDF_SEG(tile0), seg_n = PSDF_SEG(n);
        const int n = (tile - seg_tile0) * kTile + row;              // row inside its sample set
        const bool valid = n < seg_n;
        const float* __restrict__ pos = PSDF_SEG(pos);
        const float* __restrict__ g_sdf = PSDF_SEG(g_sdf);
        const float* __restrict__ g_grad = PSDF_SEG(g_grad);
        const float* __restrict__ g_geom = PSDF_SEG(g_geom);
#undef PSDF_SEG
        float x[D], v[3];
#pragma unroll
        for (int i = 0; i < D; i++) {
            x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;
            if (i < 3) v[i] = (valid && g_grad) ? g_grad[(size_t)n * 3 + i] : 0.0f;
        }
        if (g_geom) {
            // the tile's rows of the upstream geometric-feature gradient are contiguous: copy them with coalesced loads now (consumed by
            // the seed phase, several barriers later) instead of 16 scalar loads per thread 128 bytes apart (5 % of the stall samples)
            const int gw = P.g.N[3] - 1;
            const int row0 = (tile - seg_tile0) * kTile;
            const int cnt = min(kTile, seg_n - row0) * gw;
            const float* __restrict__ src = g_geom + (size_t)row0 * gw;
            for (int i = tid; i < cnt; i += kBwdThreads) s_seed[(i / gw) * (gw | 1) + (i % gw)] = src[i];
        }
        // ---------------- 1. encoder -> X: operand cores grp, grp+4, ... (4 levels = 8 features = one 16-byte core row)
        for (int kc = grp; kc < K0 / 8; kc += kGroups) {
            float fv[8], ft[1][8];
            if (kc < level_cores) {
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int l = kc * 4 + q;
                    // directional tangent along v: the barycentric weights' tangent dB_r applied to the same vertex values
                    float dcf[D], db[D + 2];
#pragma unroll
                    for (int i = 0; i < D; i++) dcf[i] = i < 3 ? v[i] * lc->scale[l * 4 + i] : 0.0f;
                    Simplex<D> s;
                    float2 val[D + 1];
                    const float2 a = level_features<D>(x, lc, l, lattice, P.T, P.cap_mask, s, val);
                    bary_tangent<D>(dcf, s, db);
                    const float w = lc->window[l];
                    float t0 = 0.f, t1 = 0.f;
#pragma unroll
                    for (int r = 0; r <= D; r++) { const float cr = db[r] * w; t0 = fmaf(val[r].x, cr, t0); t1 = fmaf(val[r].y, cr, t1); }
                    fv[2 * q] = a.x; fv[2 * q + 1] = a.y; ft[0][2 * q] = t0; ft[0][2 * q + 1] = t1;
                }
            } else {
                concat_core<1, D>(P, kc, x, &v, fv, ft);
            }
            store8(s_X, s_X + kATileBytes, row, kc, fv);
            store8(s_X + 2 * kATileBytes, s_X + 3 * kATileBytes, row, kc, ft[0]);
        }

        PSDF_PHASE(kPhEncoder);
        // ---------------- 2. forward recompute, layers 0..2. Warpgroup (mh, nh) = (wgi & 1, wgi >> 1) forms rows 64 mh .. 64 mh + 63 x column
        // half nh of both streams in its registers and consumes them in place: a_{l+1} | ta_{l+1} -> the next operand set, and the raw
        // z_{l+1} | tz_{l+1} -> accumulator columns l * 128 (l = 0, 1) or the work columns (l = 2) for the reverse sweep
        float g1[16], g2t[16];                 // gelu'(z_3), gelu''(z_3) tz_3 of this thread's chunk: consumed by the first reverse step
        float seed[2][8];                      // upstream gradient columns of this thread (prefetched before the layer-2 MMAs)
#pragma unroll 1
        for (int l = 0; l < 3; l++) {
            if (l == 1 && tid == 0) umma::bulk_wait_read0();   // X is overwritten by this layer's epilogue: the store must have read it
            umma::fence_async_smem();
            __syncthreads();
            const uint8_t* at = (l == 1) ? s_Y : s_X;
            uint8_t* dst = (l == 1) ? s_X : s_Y;
            const uint32_t col = (l == 2) ? kColWork : (uint32_t)(l * 128);
            if (l == 0 && tid == 0) {          // a_0 | ta_0 leave as they are (needed again for dW_0 at the end of the reverse sweep)
                umma::bulk_s2g(out.a0_spill + (size_t)tile * kSetBytes, s_X, kSetBytes);
                umma::bulk_commit();
            }
            if (l == 2) {                      // zbar_4 = [g_sdf, g_geom...] columns of this thread, loaded while the MMAs run
                const int Np = P.g.Np[3], nout = P.g.N[3];
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int c = grp + j * kGroups;
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const int colz = c * 8 + i;
                        float vz = 0.f;
                        if (valid && c < Np / 8) {
                            if (colz == 0) vz = g_sdf ? g_sdf[n] : 0.f;
                            else if (colz < nout) vz = g_geom ? s_seed[row * ((nout - 1) | 1) + colz - 1] : 0.f;
                        }
                        seed[j][i] = vz;
                    }
                }
            }
            const int mh = wgi & 1;
            int n0, nn;
            split_n(P.g.Np[l], wgi >> 1, n0, nn);
            float acc[2][16];
#pragma unroll
            for (int i = 0; i < 16; i++) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
            const uint32_t ro = (uint32_t)(mh * 8 * kSBO_A);
            if (nn == 32) streams_product<32, 2>(acc[0], at, 2 * kATileBytes, kATileBytes, ro, s_w + P.g.w_hi[l], s_w + P.g.w_lo[l], P.g.Kp[l], n0);
            else if (nn == 16) streams_product<16, 2>(acc[0], at, 2 * kATileBytes, kATileBytes, ro, s_w + P.g.w_hi[l], s_w + P.g.w_lo[l], P.g.Kp[l], n0);
            const float* bias = reinterpret_cast<const float*>(s_w + P.g.bias[l]);
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (8 * j < nn) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int r = frag_row(mh, h), c = n0 + frag_col(j);
                        const float z[2] = {acc[0][4 * j + 2 * h], acc[0][4 * j + 2 * h + 1]}, tz[2] = {acc[1][4 * j + 2 * h], acc[1][4 * j + 2 * h + 1]};
                        float* zp = umma::acc_ptr((uint32_t)r, col + (uint32_t)c);
                        *reinterpret_cast<float2*>(zp) = make_float2(z[0], z[1]);
                        *reinterpret_cast<float2*>(zp + 64) = make_float2(tz[0], tz[1]);
                        float a[2], ta[2];
#pragma unroll
                        for (int b = 0; b < 2; b++) {
                            const float zz = z[b] + bias[c + b];
                            const GeluEval ge = gelu_eval(zz);
                            a[b] = zz * ge.cdf;
                            ta[b] = fmaf(zz, ge.pdf, ge.cdf) * tz[b];
                        }
                        store_pair(dst, dst + kATileBytes, r, c, a[0], a[1]);
                        store_pair(dst + 2 * kATileBytes, dst + 3 * kATileBytes, r, c, ta[0], ta[1]);
                    }
                }
            }
        }
        // every layer-2 product has completed (a_2 in X is dead) and z_3 | tz_3 are stored: the GELU' / GELU'' factors of the first
        // reverse step, in the per-row layout of the reverse epilogues
        __syncthreads();
        if (grp < P.g.Np[2] / 16) {
            float z[16], tz[16];
            umma::tmem_ld16(tlane + kColWork + grp * 16, z);
            umma::tmem_ld16(tlane + kColWork + 64 + grp * 16, tz);
            activations16(z, tz, reinterpret_cast<const float*>(s_w + P.g.bias[2]) + grp * 16, g1, g2t);
        }
        PSDF_PHASE(kPhForward);
        // ---------------- 3. seed: zbar_4 = upstream gradient, tzbar_4 = e_0 -> X
        {
            const int Np = P.g.Np[3];
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int c = grp + j * kGroups;
                if (c < Np / 8) {
                    float tb[8];
#pragma unroll
                    for (int i = 0; i < 8; i++) tb[i] = (valid && c == 0 && i == 0) ? 1.0f : 0.0f;
                    store8(s_X, s_X + kATileBytes, row, c, seed[j]);
                    store8(s_X + 2 * kATileBytes, s_X + 3 * kATileBytes, row, c, tb);
                    float z16[16];
#pragma unroll
                    for (int i = 0; i < 8; i++) { z16[i] = seed[j][i]; z16[i + 8] = 0.f; }
                    int colb;
                    const float cs = colsum16(z16, lane, colb);                       // bias gradient of the output layer
                    if (!(lane & 1) && colb < 8) {
                        if (det) fx_add(&s_gb[3 * 64 + c * 8 + colb], cs);
                        else atomicAdd(&s_gbf[3 * 64 + c * 8 + colb], cs);
                    }
                }
            }
        }
        PSDF_PHASE(kPhSeed);
        // ---------------- 4. reverse sweep, layers 3..0: X = zbar_{l+1} | tzbar_{l+1}, Y = a_l | ta_l
#pragma unroll 1
        for (int l = 3; l >= 0; l--) {
            const uint32_t dw_col = tmem_base + kColDw + (uint32_t)(l >> 1) * 64 + ((l & 1) ? (16u << 16) : 0u);
            umma::fence_async_smem();
            __syncthreads();
            if (gemm_issuer) {
                const int s = wgi;
                issue_reverse(tmem_base + kColWork + s * 64, s_X + s * 2 * kATileBytes, s_X + s * 2 * kATileBytes + kATileBytes,
                              s_w + P.g.w_hi[l], s_w + P.g.w_lo[l], P.g.Kp[l], P.g.Np[l]);
                umma::mbar_arrive(&bars[1]);
            }
            if (dw_issuer && (l == 3 || l == 0)) {
                // l = 3: a_3 | ta_3 are in Y since the forward epilogue; l = 0: a_0 | ta_0 come back by TMA (requested after the
                // previous step released Y)
                if (l == 0) umma::mbar_wait(&bars[0], ld_phase);
                int n0, nn;
                split_n(P.g.Kp[l], wgi - 2, n0, nn);
                issue_dw_part(dw_col, s_X, s_Y, n0, nn, first_tile);
                umma::mbar_arrive(&bars[2]);
            }
            if (l == 1 || l == 2) {
                // beside the reverse MMAs: rebuild a_l | ta_l -> Y and the GELU' / GELU'' factors from the stored z_l, tz_l
                const int c = grp;
                if (c < P.g.Kp[l] / 16) {
                    float z[16], tz[16];
                    const uint32_t col = (uint32_t)((l - 1) * 128);
                    umma::tmem_ld16(tlane + col + c * 16, z);
                    umma::tmem_ld16(tlane + col + 64 + c * 16, tz);
                    activations16(z, tz, reinterpret_cast<const float*>(s_w + P.g.bias[l - 1]) + c * 16, g1, g2t);
                    store_set16(s_Y, row, c, z, tz);
                }
                umma::fence_async_smem();
                __syncthreads();
                if (dw_issuer) {
                    int n0, nn;
                    split_n(P.g.Kp[l], wgi - 2, n0, nn);
                    issue_dw_part(dw_col, s_X, s_Y, n0, nn, first_tile);
                    umma::mbar_arrive(&bars[2]);
                }
            }
            umma::mbar_wait(&bars[1], mma_phase);
            mma_phase ^= 1;
            const int c = grp;
            const bool have = c < P.g.Kp[l] / 16;
            float ab[16], tab_[16];
            if (have) {
                umma::tmem_ld16(tlane + kColWork + c * 16, ab);
                umma::tmem_ld16(tlane + kColWork + 64 + c * 16, tab_);
                if (l > 0) {
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const float zb = g1[i] * ab[i] + g2t[i] * tab_[i];
                        tab_[i] = g1[i] * tab_[i];
                        ab[i] = zb;                  // ab = zbar_l, tab_ = tzbar_l
                    }
                }
            }
            // X and Y are still operands of the weight-gradient MMAs
            umma::mbar_wait(&bars[2], dw_phase);
            dw_phase ^= 1;
            if (l == 1 && tid == 0) {          // Y is free: bring a_0 | ta_0 back for the last step (the store completed long ago)
                umma::bulk_wait0();
                umma::mbar_expect_tx(&bars[0], (uint32_t)kSetBytes);
                umma::bulk_g2s(s_Y, out.a0_spill + (size_t)tile * kSetBytes, (uint32_t)kSetBytes, &bars[0]);
            }
            if (l > 0) {
                if (have) {
                    store_set16(s_X, row, c, ab, tab_);
                    if (!valid) {
#pragma unroll
                        for (int i = 0; i < 16; i++) ab[i] = 0.f;
                    }
                    int colb;
                    const float cs = colsum16(ab, lane, colb);       // bias gradient: column sums over the warp's 32 rows
                    if (!(lane & 1)) {
                        if (det) fx_add(&s_gb[(l - 1) * 64 + c * 16 + colb], cs);
                        else atomicAdd(&s_gbf[(l - 1) * 64 + c * 16 + colb], cs);
                    }
                }
            } else if (have) {
                // abar_0 | tabar_0 of this row's levels (columns 2 l, 2 l + 1) -> the exchange region, for k_sdf_lattice_scatter
                float4* dst = out.xch + (size_t)tile * kTile + row;
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const int lv = c * 8 + i;
                    if (lv < P.L) dst[(size_t)lv * out.xch_stride] = make_float4(ab[2 * i], ab[2 * i + 1], tab_[2 * i], tab_[2 * i + 1]);
                }
            }
            PSDF_PHASE(kPhReverse3 + (3 - l));
        }
        ld_phase ^= 1;
        // no barrier before the next tile: every thread has waited for this tile's last MMAs (bars[1], bars[2]), the only readers of
        // X and Y, and the accumulator columns read above are rewritten only after the next tile's first __syncthreads
        if (out.phase_cycles && tid == 0) atomicAdd(out.phase_cycles + kPhTiles, 1ull);
    }
    // ---------------- weight gradients of this CTA: accumulators -> global (+=). Warp w reads lanes 32 (w & 3) .. +31 of column chunk w >> 2:
    // lanes 0..15 hold rows 16 (w & 3) + lane of the even layer of the pair, lanes 16..31 the same rows of the odd layer
    if (!first_tile) {
        const int q = warp & 3, c = warp >> 2;
#pragma unroll 1
        for (int p = 0; p < 2; p++) {
            float acc[16];
            umma::tmem_ld16(tlane + kColDw + p * 64 + c * 16, acc);
            const int l = 2 * p + (lane >> 4), m = q * 16 + (lane & 15);
            if (m < P.g.N[l] && det) {
                const int K = P.g.K[l];
                unsigned long long* dst = out.fx_mlp + l * kFxW + m * K;
#pragma unroll
                for (int i = 0; i < 16; i++) if (c * 16 + i < K) fx_add(dst + c * 16 + i, acc[i]);
            } else if (m < P.g.N[l]) {
                const int K = P.g.K[l];
                float* dst = out.gW[l] + (size_t)m * K + c * 16;
                const bool vec = (K & 3) == 0 && ((uintptr_t)out.gW[l] & 15) == 0;      // rows stay 16-byte aligned
#pragma unroll
                for (int i = 0; i < 16; i += 4) {
                    const int k = c * 16 + i;
                    if (vec && k + 3 < K) red_v4(dst + i, acc[i], acc[i + 1], acc[i + 2], acc[i + 3]);
                    else {
#pragma unroll
                        for (int j = 0; j < 4; j++) if (k + j < K) atomicAdd(dst + i + j, acc[i + j]);
                    }
                }
            }
        }
    }
    for (int i = tid; i < kNL * 64; i += kBwdThreads) {
        int l = i >> 6, c = i & 63;
        if (det) { if (c < P.g.N[l] && s_gb[i] != 0ull) atomicAdd(out.fx_mlp + kFxB + l * 64 + c, s_gb[i]); }
        else if (c < P.g.N[l] && s_gbf[i] != 0.0f) atomicAdd(out.gbias[l] + c, s_gbf[i]);
    }
    PSDF_PHASE(kPhFlush);
    if (tid == 0) umma::bulk_wait0();      // spill stores complete before the CTA retires
}

// Encoder backward: lattice[l][idx_r] += window_l (B_r abar_0[l] + dB_r tabar_0[l]) from the exchange rows of k_sdf_fused_backward.
// blockIdx.y = level (blocks of one level run together: its table of gradient accumulators stays in L2 while they land), warp =
// 32 consecutive sample slots, i.e. the rows of one warp of the persistent kernel. The simplex and the barycentric tangent are
// recomputed from the positions and upstream gradients.
constexpr int kScatterThreads = 256;
template <int D>
__global__ void __launch_bounds__(kScatterThreads, 8)
k_sdf_lattice_scatter(FusedParams P, Segments S, const float4* __restrict__ xch, int xch_stride, const float* __restrict__ scale,
                      const float* __restrict__ shift, const float* __restrict__ window, float* __restrict__ grad_lattice,
                      unsigned long long* __restrict__ fx_lattice) {
    const int slot = blockIdx.x * kScatterThreads + threadIdx.x;      // tile * 128 + row
    if (slot >= xch_stride) return;                                  // whole warps (xch_stride % 128 == 0)
    const int l = blockIdx.y, lane = threadIdx.x & 31, tile = slot / kTile;
    const int seg = tile >= S.tile0[2] ? 2 : (tile >= S.tile0[1] ? 1 : 0);
#define PSDF_SEG(f) (seg == 2 ? S.f[2] : (seg == 1 ? S.f[1] : S.f[0]))
    const int n = (tile - PSDF_SEG(tile0)) * kTile + (slot % kTile);
    const bool valid = n < PSDF_SEG(n);
    const float* __restrict__ pos = PSDF_SEG(pos);
    const float* __restrict__ g_grad = PSDF_SEG(g_grad);
#undef PSDF_SEG
    float x[D], v[D], sc[D], sh[D];
#pragma unroll
    for (int i = 0; i < D; i++) {
        x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;
        v[i] = (i < 3 && valid && g_grad) ? g_grad[(size_t)n * 3 + i] : 0.0f;
        sc[i] = scale[l * D + i];
        sh[i] = shift ? shift[l * D + i] : 0.0f;
    }
    const float w = window ? window[l] : 1.0f;
    const float4 a = xch[(size_t)l * xch_stride + slot];
    const bool aggregate = sc[0] < kAggregateBelowScale && !(P.knockout & 2);      // warp-uniform (l is)
    const bool do_red = !(P.knockout & 1);            // diagnostics (PSDF_EXPERIMENT_KNOCKOUT): bit 0 no atomics, bit 1 no aggregation
    scatter_level<true, D>(x, v, sc, sh, w, a.x, a.y, a.z, a.w, valid, aggregate, do_red, lane, P.cap_mask, (unsigned)P.T,
                  grad_lattice + (size_t)l * P.T * 2, fx_lattice ? fx_lattice + (size_t)l * P.T * 2 : nullptr);
}

// workspace per 128-sample tile: the encoder operand tiles (a_0 | ta_0, 64 KB), written by TMA store in the forward recompute and read
// back by the same CTA for the first layer's weight gradient, and the exchange rows abar_0 | tabar_0 (16 bytes per sample and level,
// sized for kMaxLevels so that the size depends on the sample count alone)
constexpr long long kWsTileBytes = kSetBytes + (long long)kTile * kMaxLevels * sizeof(float4);

#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {

long long psdf_sdf_fused_backward_workspace_bytes(int N) {
    const int ntiles = div_up(N > 0 ? N : 1, kTile);
    return (long long)ntiles * kWsTileBytes;
}

}  // extern "C"

template <int D>
static int launch_backward(int nseg, const int* Ns, const float* const* pos, const float* const* g_sdf, const float* const* g_grad,
                           const float* const* g_geom, int L, int T, const float* lattice, const float* scale_factor, const float* shift,
                           const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, float* grad_lattice,
                           uint8_t* workspace, float* const* gW, float* const* gb, void* stream) {
    if (nseg < 1 || nseg > kMaxSeg || L < 4 || L > kMaxLevels || (L % 4) != 0 || hidden > 64 || hidden % 16 != 0 || out_dim > 64) return PSDF_ERR_UNSUPPORTED;
    FusedParams P;
    P.L = L; P.T = T;
    P.cap_mask = t_magic(T);
    P.points_scaling = points_scaling;
    P.in_dim = (L + 2) * 2;
    if (P.in_dim > 64) return PSDF_ERR_UNSUPPORTED;
    P.g = make_geom(P.in_dim, hidden, out_dim);
    static const int knockout = getenv("PSDF_EXPERIMENT_KNOCKOUT") ? atoi(getenv("PSDF_EXPERIMENT_KNOCKOUT")) : 0;
    P.knockout = knockout;
    Segments S;
    int tiles = 0, total = 0;
    for (int i = 0; i < kMaxSeg; i++) {
        const int n = i < nseg ? Ns[i] : 0;
        if (n < 0) return PSDF_ERR_ARG;
        S.n[i] = n; S.tile0[i] = tiles;
        S.pos[i] = i < nseg ? pos[i] : nullptr; S.g_sdf[i] = i < nseg ? g_sdf[i] : nullptr;
        S.g_grad[i] = i < nseg ? g_grad[i] : nullptr; S.g_geom[i] = i < nseg ? g_geom[i] : nullptr;
        tiles += div_up(n, kTile);
        total += n;
    }
    S.tile0[kMaxSeg] = tiles;
    P.N = total;
    if (tiles == 0) return PSDF_OK;
    const DetBufs* dbuf = det_buffers();
    if (dbuf && (long long)L * T * 2 > dbuf->lattice_len) return PSDF_ERR_UNSUPPORTED;   // reserve more with psdf_set_deterministic
    BwdOut out;
    for (int l = 0; l < kNL; l++) { out.gW[l] = gW[l]; out.gbias[l] = gb[l]; }
    out.fx_mlp = dbuf ? dbuf->sdf_mlp : nullptr;
    out.a0_spill = workspace;
    out.xch = reinterpret_cast<float4*>(workspace + (size_t)tiles * kSetBytes);
    out.xch_stride = tiles * kTile;
    // diagnostics: PSDF_PHASE_TIMING=1 prints thread 0's clock64 breakdown per phase (average cycles per tile) after every launch
    static const bool timing = getenv("PSDF_PHASE_TIMING") && atoi(getenv("PSDF_PHASE_TIMING")) != 0;
    static unsigned long long* d_cycles = nullptr;
    static cudaEvent_t ev[3];
    out.phase_cycles = nullptr;
    if (timing) {
        if (!d_cycles) {
            cudaMalloc(&d_cycles, 16 * sizeof(unsigned long long));
            for (auto& e : ev) cudaEventCreate(&e);
        }
        cudaMemsetAsync(d_cycles, 0, 16 * sizeof(unsigned long long), ST);
        out.phase_cycles = d_cycles;
        cudaEventRecord(ev[0], ST);
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = (size_t)P.g.total + 2 * kSetBytes + sizeof(LevelC) + kNL * 64 * sizeof(unsigned long long) + 64 + (size_t)kTile * (size_t)((out_dim - 1) | 1) * sizeof(float);
    if (smem > 227 * 1024) return PSDF_ERR_UNSUPPORTED;
    { static bool optin_[64]; psdf::psdf_optin_smem(k_sdf_fused_backward<D>, 227 * 1024, optin_); }
    k_sdf_fused_backward<D><<<min(min(tiles, sms), kAccCtas), kBwdThreads, smem, ST>>>(P, S, reinterpret_cast<const float2*>(lattice), scale_factor, shift, window,
                                                                    blob, out);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[1], ST);
    k_sdf_lattice_scatter<D><<<dim3(div_up(out.xch_stride, kScatterThreads), L), kScatterThreads, 0, ST>>>(
        P, S, out.xch, out.xch_stride, scale_factor, shift, window, grad_lattice, dbuf ? dbuf->sdf_lattice : nullptr);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[2], ST);
    if (dbuf) {      // deterministic mode: fixed-point totals -> the float gradients (+=)
        FxSegs F;
        F.add(dbuf->sdf_lattice, grad_lattice, (long long)L * T * 2);
        for (int l = 0; l < kNL; l++) {
            F.add(dbuf->sdf_mlp + l * kFxW, gW[l], (long long)P.g.N[l] * P.g.K[l]);
            F.add(dbuf->sdf_mlp + kFxB + l * 64, gb[l], P.g.N[l]);
        }
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    if (timing) {
        unsigned long long h[16];
        cudaMemcpyAsync(h, d_cycles, sizeof(h), cudaMemcpyDeviceToHost, ST);
        cudaStreamSynchronize(ST);
        const double t = h[kPhTiles] ? (double)h[kPhTiles] : 1.0;
        float ms_fused = 0.f, ms_scatter = 0.f;
        cudaEventElapsedTime(&ms_fused, ev[0], ev[1]);
        cudaEventElapsedTime(&ms_scatter, ev[1], ev[2]);
        fprintf(stderr, "[psdf_sdf_fused_backward N=%d tiles=%llu] cycles/tile: encoder %.0f forward %.0f seed %.0f rev3 %.0f rev2 %.0f rev1 %.0f rev0 %.0f "
                        "| flush/CTA %.0f | fused kernel %.3f ms, lattice scatter %.3f ms\n", total, h[kPhTiles], h[0] / t, h[1] / t, h[2] / t, h[3] / t,
                h[4] / t, h[5] / t, h[6] / t, (double)h[kPhFlush] / min(tiles, sms), ms_fused, ms_scatter);
    }
    return PSDF_OK;
}

extern "C" {

// workspace of a multi-set launch: every set is padded to whole tiles
long long psdf_sdf_fused_backward_multi_workspace_bytes(int N0, int N1, int N2) {
    return (long long)(div_up(N0 > 0 ? N0 : 0, kTile) + div_up(N1 > 0 ? N1 : 0, kTile) + div_up(N2 > 0 ? N2 : 0, kTile) + 1) * kWsTileBytes;
}

// grad_lattice, grad_W_l [N_l, K_l] and grad_bias_l are accumulated (+=).
int psdf_sdf_fused_backward(int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor, const float* shift,
                            const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, const float* g_sdf,
                            const float* g_grad, const float* g_geom, float* grad_lattice, uint8_t* workspace, float* gW0, float* gW1,
                            float* gW2, float* gW3, float* gb0, float* gb1, float* gb2, float* gb3, void* stream) {
    if (N < 0) return PSDF_ERR_ARG;
    if (N == 0) return PSDF_OK;
    float* gW[kNL] = {gW0, gW1, gW2, gW3};
    float* gb[kNL] = {gb0, gb1, gb2, gb3};
    return launch_backward<3>(1, &N, &pos, &g_sdf, &g_grad, &g_geom, L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob,
                           grad_lattice, workspace, gW, gb, stream);
}

// The same backward over up to three independent sample sets in ONE launch (unused sets: N = 0). Used by the training iteration to run
// the main samples, the curvature pass and the off-surface points together (each psdf_sdf_fused_forward call of the iteration has its
// own upstream gradients; the parameters, hence the accumulated gradients, are shared).
int psdf_sdf_fused_backward_multi(int L, int T, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                                  float points_scaling, int hidden, int out_dim, const uint8_t* blob, int N0, const float* pos0,
                                  const float* g_sdf0, const float* g_grad0, const float* g_geom0, int N1, const float* pos1,
                                  const float* g_sdf1, const float* g_grad1, const float* g_geom1, int N2, const float* pos2,
                                  const float* g_sdf2, const float* g_grad2, const float* g_geom2, float* grad_lattice, uint8_t* workspace,
                                  float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1, float* gb2, float* gb3, void* stream) {
    const int Ns[3] = {N0, N1, N2};
    const float* pos[3] = {pos0, pos1, pos2};
    const float* gs[3] = {g_sdf0, g_sdf1, g_sdf2};
    const float* gg[3] = {g_grad0, g_grad1, g_grad2};
    const float* gm[3] = {g_geom0, g_geom1, g_geom2};
    float* gW[kNL] = {gW0, gW1, gW2, gW3};
    float* gb[kNL] = {gb0, gb1, gb2, gb3};
    return launch_backward<3>(3, Ns, pos, gs, gg, gm, L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, grad_lattice,
                              workspace, gW, gb, stream);
}

// psdf_sdf_fused_backward_multi at either input width: positions [N_i, pos_dim], pos_dim 3 (psdf_sdf_fused_backward_multi) or 4 (space-time
// positions; g_grad [N_i,3] is the upstream gradient of the spatial derivatives, so the tangent direction is (g_grad, 0)). Same workspace.
int psdf_sdf_fused_backward_multi_dim(int pos_dim, int L, int T, const float* lattice, const float* scale_factor, const float* shift,
                                      const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, int N0,
                                      const float* pos0, const float* g_sdf0, const float* g_grad0, const float* g_geom0, int N1,
                                      const float* pos1, const float* g_sdf1, const float* g_grad1, const float* g_geom1, int N2,
                                      const float* pos2, const float* g_sdf2, const float* g_grad2, const float* g_geom2, float* grad_lattice,
                                      uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1, float* gb2,
                                      float* gb3, void* stream) {
    const int Ns[3] = {N0, N1, N2};
    const float* pos[3] = {pos0, pos1, pos2};
    const float* gs[3] = {g_sdf0, g_sdf1, g_sdf2};
    const float* gg[3] = {g_grad0, g_grad1, g_grad2};
    const float* gm[3] = {g_geom0, g_geom1, g_geom2};
    float* gW[kNL] = {gW0, gW1, gW2, gW3};
    float* gb[kNL] = {gb0, gb1, gb2, gb3};
    if (pos_dim == 3)
        return launch_backward<3>(3, Ns, pos, gs, gg, gm, L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob,
                                  grad_lattice, workspace, gW, gb, stream);
    if (pos_dim == 4)
        return launch_backward<4>(3, Ns, pos, gs, gg, gm, L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob,
                                  grad_lattice, workspace, gW, gb, stream);
    return PSDF_ERR_UNSUPPORTED;
}

}  // extern "C"
