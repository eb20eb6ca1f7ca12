// Training backward of the fused encoding + SDF MLP (sm_90a, wgmma): given d loss / d {sdf, d sdf/dx, geom}
// per sample it produces the lattice gradient, the bias gradients and the weight gradients. Four kernels: a kernel with many warps per SM
// builds the layer-0 operand tiles a_0 | ta_0 of every tile (k_sdf_input_tiles); the persistent tensor-core kernel loads them by TMA,
// forms the weight-gradient products from the operand tiles while they are still in shared memory (summed over all tiles of the CTA,
// left in a slab per CTA that k_dw_reduce adds up) and hands abar_0 | tabar_0 to a full-occupancy kernel that scatters them into the
// lattice gradient.
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
// Per 128-sample tile (512 threads: row = tid & 127, group g = tid >> 7 owns operand cores g, g+4, .. in the seed phase). Every
// product lands in the registers of the warpgroup that issues it: warpgroup (mh, nh) = (wgi & 1, wgi >> 1) forms rows
// 64 mh .. 64 mh + 63 x column half nh (split_n) of both streams, the value and the tangent of one (row, column) in the same thread, and
// consumes them in place. Two 64 KB operand-tile buffers X, Y ([value hi | value lo | tangent hi | tangent lo]):
//   1. tile load: a_0 | ta_0 -> X by ONE TMA load (64 KB / tile, written by k_sdf_input_tiles and re-read from L2 in step 4). The next
//      tile's load is issued as soon as the step-0 products have read X, so it lands behind the exchange stores and the loop turnaround
//   2. forward recompute, layers 0..2: a_1 -> Y, a_2 -> X, a_3 -> Y straight from the fragments; the raw z_1, z_2 (value + tangent)
//      go to this thread's slots of the CTA's stash (global, L2 resident) and come back to the same thread in the reverse sweep: the
//      reverse step l splits its Kp_l = Np_{l-1} columns exactly as the forward layer l-1 split them, so it needs no barrier.
//      gelu'(z_3), gelu''(z_3) tz_3 stay in registers (layer 3 is reversed right away)
//   3. seed zbar_4 -> X
//   4. reverse sweep l = 3..0, one wgmma group per warpgroup:  abar_l | tabar_l = zbar_{l+1} | tzbar_{l+1} W_l uses the FORWARD
//      weight tile as an MN-major B operand (no transposed copy, weights resident for the CTA's lifetime), and columns
//      16 wgi .. 16 wgi + 15 of dW_l += zbar_{l+1}^T a_l + tzbar_{l+1}^T ta_l (M = 64) as one register chain over both streams: the sample
//      axis is the MMA K dimension and a K-major operand tile IS an MN-major operand for that product, so X and Y are multiplied
//      as they sit. The CTA's dW sums live in the stash between tiles (one read-modify-write per layer and tile, same thread).
//      After a barrier the fragments become zbar_l | tzbar_l -> X, the bias gradient (column sums over each 32-row group: the odd
//      warp's fragments through shared memory, then the thread's two rows, then shuffles, in exactly the order of colsum16 over the
//      rows of one warp in the per-row layout, so the partial sums and their one fixed-point rounding per tile, column and 32 rows
//      have the bits of the per-row sum),
//      and a_{l-1} | ta_{l-1} are rebuilt into Y from the stashed z_{l-1} (l = 3, 2) or come back by TMA (l = 1).
//      In the last step (l = 0) abar_0 | tabar_0 leave from the registers to the exchange region of the workspace, one float4
//      (a0, a1, t0, t1) per level and sample, [level][sample slot]: a thread's column pair is one level.
// The encoder forward is its own launch, k_sdf_input_tiles: inside the persistent kernel its dependent lattice gathers ran on 16 warps
// per SM with the tensor cores idle; on its own it runs with 40 (D = 3) or 32 (D = 4) warps per SM.
// The encoder backward is its own launch, k_sdf_lattice_scatter: warp-aggregated red.global.add.v2.f32 into the lattice gradient.
// Inside the persistent kernel it was the longest phase of a tile (one CTA of 16 warps per SM, tensor cores idle, long dependent chains
// of simplex recompute, match_any, shuffle sums and reductions); on its own it runs with every warp slot of the SM occupied. Its warps
// are the rows of the persistent kernel's warps, so the match_any groups and the float peer sums are the same.
// Deterministic mode (common.cuh): every gradient (lattice, weights, biases) is summed in fixed point instead and added to the float
// gradients by the flush that follows the launches.
// Stash of a CTA (float4 slots, slot index * 512 + tid): [0,16) z_1 | tz_1, z_2 | tz_2 fragments (8 slots per layer), [16,24) dW_0..dW_3
// (2 slots per layer). At the end of the kernel the dW sums go to the CTA's slab of g_dw_sdf_bwd: fx_of of the fp32 sum in
// deterministic mode (the value the per-CTA atomics added), the fp32 sum otherwise.
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include "fused_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;

namespace {
constexpr int kBwdThreads = 512;
constexpr int kGroups = kBwdThreads / kTile;
constexpr int kSetBytes = 4 * kATileBytes;         // one operand tile set [value hi | value lo | tangent hi | tangent lo]
constexpr int kStashDw = 16, kStashSlots = 24;      // stash map (float4 slots per thread), see the header
__device__ float4 g_stash_bwd[(size_t)kAccCtas * kStashSlots * kBwdThreads];     // per-CTA stashes, 192 KB each
constexpr int kFxW = kDetSdfW, kFxB = 4 * kDetSdfW;    // weight / bias offsets in DetBufs::sdf_mlp
// weight-gradient sums of each CTA, [CTA][layer][64 rows][64 columns] (k_dw_reduce): fixed point (fx_of) in deterministic mode, else
// float (the same slot indices in the float view)
constexpr int kDwLd = 64, kDwSlots = kNL * kDwLd * kDwLd;
__device__ unsigned long long g_dw_sdf_bwd[(size_t)kAccCtas * kDwSlots];
struct SdfDwSlab { static __device__ const void* get() { return g_dw_sdf_bwd; } };

struct BwdOut {
    const uint8_t* a0_spill;  // [ntiles][64 KB] layer-0 operand tiles a_0 | ta_0 (k_sdf_input_tiles)
    float4* xch;        // [L][xch_stride] abar_0 | tabar_0 (a0, a1, t0, t1) per level and sample slot (tile * 128 + row)
    int xch_stride;     // sample slots = ntiles * 128
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
enum { kPhTileLoad = 0, kPhForward = 1, kPhSeed = 2, kPhReverse3 = 3, kPhReverse2 = 4, kPhReverse1 = 5, kPhReverse0 = 6, kPhFlush = 7,
       kPhTiles = 8 };
#define PSDF_PHASE(id)                                                                     \
    do {                                                                                   \
        if (out.phase_cycles && tid == 0) {                                                \
            const long long now_ = clock64();                                              \
            atomicAdd(out.phase_cycles + (id), (unsigned long long)(now_ - phase_t0));     \
            phase_t0 = now_;                                                               \
        }                                                                                  \
    } while (0)

// zz = z + bias: a = gelu(zz), ta = gelu'(zz) tz; g1 = gelu'(zz), g2t = gelu''(zz) tz
__device__ __forceinline__ void activation(float z, float tz, float bias, float& a, float& ta, float& g1, float& g2t) {
    const float zz = z + bias;
    const GeluEval ge = gelu_eval(zz);
    const float d1 = fmaf(zz, ge.pdf, ge.cdf);
    g2t = ge.pdf * (2.0f - zz * zz) * tz;
    a = zz * ge.cdf;
    ta = d1 * tz;
    g1 = d1;
}

// columns [n0, n0 + 16) of  dW (+)= zbar^T a + tzbar^T ta  into the issuing warpgroup's registers (M = 64, umma::wg_mma_regs fragments):
// both tile sets consumed as MN-major operands, K = the 128 samples, the value stream then the tangent stream in one chain. Issue only.
__device__ __forceinline__ void issue_dw16(float* d, const uint8_t* zset, const uint8_t* aset, int n0, bool accumulate) {
    const uint32_t aoff = (n0 / 8) * kLBO;
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const uint64_t dzh = umma::make_desc(umma::smem_u32(zset + s * 2 * kATileBytes), kSBO_A, kLBO);
        const uint64_t dzl = umma::make_desc(umma::smem_u32(zset + s * 2 * kATileBytes + kATileBytes), kSBO_A, kLBO);
        const uint64_t dah = umma::make_desc(umma::smem_u32(aset + s * 2 * kATileBytes) + aoff, kSBO_A, kLBO);
        const uint64_t dal = umma::make_desc(umma::smem_u32(aset + s * 2 * kATileBytes + kATileBytes) + aoff, kSBO_A, kLBO);
        // 16 samples = two 8-sample groups per K step
        umma::wg_mma_regs<16, 1, 1>(d, dzh, dzl, dah, dal, (2 * kSBO_A) >> 4, (2 * kSBO_A) >> 4, kTile / 16, accumulate || s > 0);
    }
}

// Layer-0 operand tiles a_0 | ta_0 of every tile of the launch -> a0_spill ([tile][64 KB], the bytes of X in the persistent kernel):
// the window-weighted features of each level and their directional tangent along v (the barycentric weights' tangent dB_r applied to
// the same vertex values), then the concatenated points. Thread (tile, operand core kc, row): a warp is 32 consecutive rows of one
// core (4 levels = 8 features = one 16-byte core row), as in the persistent kernel's encoder phase that this replaces, so its gathers
// are the same. Invalid rows (past the end of their sample set) are built from x = v = 0. Cores past Kp[0] are not written.
// D = 3: positions [N,3]; D = 4: space-time positions [N,4] with the tangent along (g_grad, 0) (g_grad holds spatial derivatives)
constexpr int kInputTileThreads = 256;
template <int D>
__global__ void __launch_bounds__(kInputTileThreads)
k_sdf_input_tiles(FusedParams P, Segments S, const float2* __restrict__ lattice, const float* __restrict__ scale,
                  const float* __restrict__ shift, const float* __restrict__ window, uint8_t* __restrict__ a0_spill) {
    __shared__ LevelC lc;
    load_level_consts<D>(&lc, P.L, scale, shift, window, threadIdx.x, kInputTileThreads);
    __syncthreads();
    const int cores = P.g.Kp[0] / 8, level_cores = P.L / 4;
    const int u = blockIdx.x * kInputTileThreads + threadIdx.x;          // (tile * cores + kc) * 128 + row
    const int row = u % kTile, kc = (u / kTile) % cores, tile = u / (kTile * cores);
    if (tile >= S.tile0[kMaxSeg]) return;
    const int seg = tile >= S.tile0[2] ? 2 : (tile >= S.tile0[1] ? 1 : 0);
#define PSDF_SEG(f) (seg == 2 ? S.f[2] : (seg == 1 ? S.f[1] : S.f[0]))     // no dynamic indexing of the parameter struct (local-memory copy)
    const int n = (tile - PSDF_SEG(tile0)) * kTile + row;              // row inside its sample set
    const bool valid = n < PSDF_SEG(n);
    const float* __restrict__ pos = PSDF_SEG(pos);
    const float* __restrict__ g_grad = PSDF_SEG(g_grad);
#undef PSDF_SEG
    float x[D], v[3];
#pragma unroll
    for (int i = 0; i < D; i++) {
        x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;
        if (i < 3) v[i] = (valid && g_grad) ? g_grad[(size_t)n * 3 + i] : 0.0f;
    }
    float fv[8], ft[1][8];
    if (kc < level_cores) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int l = kc * 4 + q;
            float dcf[D], db[D + 2];
#pragma unroll
            for (int i = 0; i < D; i++) dcf[i] = i < 3 ? v[i] * lc.scale[l * 4 + i] : 0.0f;
            Simplex<D> s;
            float2 val[D + 1];
            const float2 a = level_features<D>(x, &lc, l, lattice, P.T, P.cap_mask, s, val);
            bary_tangent<D>(dcf, s, db);
            const float w = lc.window[l];
            float t0 = 0.f, t1 = 0.f;
#pragma unroll
            for (int r = 0; r <= D; r++) { const float cr = db[r] * w; t0 = fmaf(val[r].x, cr, t0); t1 = fmaf(val[r].y, cr, t1); }
            fv[2 * q] = a.x; fv[2 * q + 1] = a.y; ft[0][2 * q] = t0; ft[0][2 * q + 1] = t1;
        }
    } else {
        concat_core<1, D>(P, kc, x, &v, fv, ft);
    }
    uint8_t* t = a0_spill + (size_t)tile * kSetBytes;
    store8(t, t + kATileBytes, row, kc, fv);
    store8(t + 2 * kATileBytes, t + 3 * kATileBytes, row, kc, ft[0]);
}

// The same code at D = 3 and 4 (the input width only matters to k_sdf_input_tiles and the scatter); one instantiation per width
template <int D>
__global__ void __launch_bounds__(kBwdThreads, 1)
k_sdf_fused_backward(FusedParams P, Segments S, const uint8_t* __restrict__ blob, BwdOut out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_w = smem;                                   // forward operand blob (weights hi/lo + biases), resident
    uint8_t* s_X = smem + P.g.total;
    uint8_t* s_Y = s_X + kSetBytes;
    // 4 x 64 bias-gradient accumulators of this CTA: float (s_gbf), or fixed point (s_gb) in deterministic mode
    unsigned long long* s_gb = reinterpret_cast<unsigned long long*>(s_Y + kSetBytes);
    float* s_gbf = reinterpret_cast<float*>(s_gb);
    const bool det = out.fx_mlp != nullptr;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gb + kNL * 64);   // [0] weights, a_0 | ta_0 reload into Y; [1] tile loads into X
    float* s_seed = reinterpret_cast<float*>(bars + 5);   // [128][(out_dim - 1) | 1] upstream d loss / d geom of the tile (coalesced copy)
    // the same bytes in the reverse sweep (s_seed is dead from the seed phase to the next tile): [8 warp pairs][16][32 lanes] the odd
    // warp's zbar fragments for the bias column sums
    float* s_bx = s_seed;

    const int tid = threadIdx.x, warp = warp_uniform(tid >> 5), lane = tid & 31;
    const int row = tid & 127, grp = tid >> 7;
    const int wgi = warp >> 2, mh = wgi & 1, nh = wgi >> 1;
    float4* stash = g_stash_bwd + (size_t)blockIdx.x * kStashSlots * kBwdThreads + tid;     // this thread's slot 0

    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_init(&bars[1], 1);
        umma::mbar_fence_init();
    }
    for (int i = tid; i < kNL * 64; i += kBwdThreads) s_gb[i] = 0ull;     // also clears s_gbf
    __syncthreads();
    const int ntiles = S.tile0[kMaxSeg];
    if (tid == 0) {          // the weights and the first tile (the grid has no more CTAs than tiles)
        umma::mbar_expect_tx(&bars[0], (uint32_t)P.g.total);
        umma::bulk_g2s(s_w, blob, (uint32_t)P.g.total, &bars[0]);
        umma::mbar_expect_tx(&bars[1], (uint32_t)kSetBytes);
        umma::bulk_g2s(s_X, out.a0_spill + (size_t)blockIdx.x * kSetBytes, (uint32_t)kSetBytes, &bars[1]);
    }
    __syncthreads();
    umma::mbar_wait(&bars[0], 0);
    uint32_t ld_phase = 1;      // parity of bars[0]'s a_0 | ta_0 reload; bars[1] (one tile load per tile) runs at ld_phase ^ 1

    bool first_tile = true;
    long long phase_t0 = out.phase_cycles ? clock64() : 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, first_tile = false) {
        const int seg = tile >= S.tile0[2] ? 2 : (tile >= S.tile0[1] ? 1 : 0);
#define PSDF_SEG(f) (seg == 2 ? S.f[2] : (seg == 1 ? S.f[1] : S.f[0]))     // no dynamic indexing of the parameter struct (local-memory copy)
        const int seg_tile0 = PSDF_SEG(tile0), seg_n = PSDF_SEG(n);
        const int n = (tile - seg_tile0) * kTile + row;              // row inside its sample set
        const bool valid = n < seg_n;
        const float* __restrict__ g_sdf = PSDF_SEG(g_sdf);
        const float* __restrict__ g_geom = PSDF_SEG(g_geom);
#undef PSDF_SEG
        if (g_geom) {
            // the tile's rows of the upstream geometric-feature gradient are contiguous: copy them with coalesced loads now (consumed by
            // the seed phase, several barriers later) instead of 16 scalar loads per thread 128 bytes apart (5 % of the stall samples)
            const int gw = P.g.N[3] - 1;
            const int row0 = (tile - seg_tile0) * kTile;
            const int cnt = min(kTile, seg_n - row0) * gw;
            const float* __restrict__ src = g_geom + (size_t)row0 * gw;
            for (int i = tid; i < cnt; i += kBwdThreads) s_seed[(i / gw) * (gw | 1) + (i % gw)] = src[i];
        }
        // ---------------- 1. a_0 | ta_0 of this tile -> X (TMA load issued next to the weight load or after the previous tile's step 0)
        umma::mbar_wait(&bars[1], ld_phase ^ 1);
        PSDF_PHASE(kPhTileLoad);
        // ---------------- 2. forward recompute, layers 0..2. Warpgroup (mh, nh) forms rows 64 mh .. 64 mh + 63 x column half nh of both
        // streams in its registers and consumes them in place: a_{l+1} | ta_{l+1} -> the next operand set, and the raw z_{l+1} | tz_{l+1}
        // -> this thread's stash slots (l = 0, 1) or the GELU' / GELU'' factors of the first reverse step (l = 2)
        float g1[16], g2t[16];                 // gelu'(z_l), gelu''(z_l) tz_l of this thread's fragments, for the reverse step l
        float seed[2][8];                      // upstream gradient columns of this thread (prefetched before the layer-2 MMAs)
#pragma unroll 1
        for (int l = 0; l < 3; l++) {
            umma::fence_async_smem();
            __syncthreads();
            const uint8_t* at = (l == 1) ? s_Y : s_X;
            uint8_t* dst = (l == 1) ? s_X : s_Y;
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
            int n0, nn;
            split_n(warp_uniform(P.g.Np[l]), nh, n0, nn);
            float acc[2][16];
#pragma unroll
            for (int i = 0; i < 16; i++) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
            const uint32_t ro = (uint32_t)(mh * 8 * kSBO_A);
            if (nn == 32) streams_product<32, 2>(acc[0], at, 2 * kATileBytes, kATileBytes, ro, s_w + warp_uniform(P.g.w_hi[l]), s_w + warp_uniform(P.g.w_lo[l]), warp_uniform(P.g.Kp[l]), n0);
            else if (nn == 16) streams_product<16, 2>(acc[0], at, 2 * kATileBytes, kATileBytes, ro, s_w + warp_uniform(P.g.w_hi[l]), s_w + warp_uniform(P.g.w_lo[l]), warp_uniform(P.g.Kp[l]), n0);
            if (l < 2) {
                // fragment block j of stream s -> slot 8 l + 4 s + j (thread-private: read back by this thread in the reverse step l + 1)
#pragma unroll
                for (int s = 0; s < 2; s++)
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (8 * j < nn) stash[(8 * l + 4 * s + j) * kBwdThreads] = make_float4(acc[s][4 * j], acc[s][4 * j + 1], acc[s][4 * j + 2], acc[s][4 * j + 3]);
            }
            const float* bias = reinterpret_cast<const float*>(s_w + warp_uniform(P.g.bias[l]));
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (8 * j < nn) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int r = frag_row(mh, h), c = n0 + frag_col(j);
                        float a[2], ta[2];
#pragma unroll
                        for (int b = 0; b < 2; b++) {
                            const int i = 4 * j + 2 * h + b;
                            float d1, d2t;
                            activation(acc[0][i], acc[1][i], bias[c + b], a[b], ta[b], d1, d2t);
                            if (l == 2) { g1[i] = d1; g2t[i] = d2t; }
                        }
                        store_pair(dst, dst + kATileBytes, r, c, a[0], a[1]);
                        store_pair(dst + 2 * kATileBytes, dst + 3 * kATileBytes, r, c, ta[0], ta[1]);
                    }
                }
            }
        }
        // every layer-2 product has completed: a_2 in X is dead
        __syncthreads();
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
        const int nbase = (tile - seg_tile0) * kTile;
        const bool rvalid0 = nbase + frag_row(mh, 0) < seg_n, rvalid1 = nbase + frag_row(mh, 1) < seg_n;   // this thread's fragment rows
#pragma unroll 1
        for (int l = 3; l >= 0; l--) {
            umma::fence_async_smem();
            __syncthreads();
            if (l == 0) umma::mbar_wait(&bars[0], ld_phase);     // a_0 | ta_0 are back in Y
            int n0, nn;
            split_n(warp_uniform(P.g.Kp[l]), nh, n0, nn);
            const bool dw = 16 * wgi < warp_uniform(P.g.Kp[l]);              // this warpgroup's 16 columns of dW_l
            float4* dws = stash + (kStashDw + 2 * l) * kBwdThreads;
            float acc[2][16], dwa[8];                          // acc[0] = abar_l, acc[1] = tabar_l; dwa: the CTA's sum of dW_l
#pragma unroll
            for (int i = 0; i < 16; i++) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
#pragma unroll
            for (int q = 0; q < 2; q++) {
                const float4 v = (dw && !first_tile) ? dws[q * kBwdThreads] : make_float4(0.f, 0.f, 0.f, 0.f);
                dwa[4 * q] = v.x; dwa[4 * q + 1] = v.y; dwa[4 * q + 2] = v.z; dwa[4 * q + 3] = v.w;
            }
            const uint32_t ro = (uint32_t)(mh * 8 * kSBO_A);
            // the reverse product (NC columns, none for NC = 0) and the dW chain as one wgmma group. Each column count is a whole group
            // of its own: a branch between the fence and the wait joins the fragments of the two paths inside the group, and those
            // register moves make ptxas serialize every wgmma chain of the kernel (C7515)
            auto products = [&](auto nc) {
                constexpr int NC = decltype(nc)::value;
                umma::wgmma_fence();
                if constexpr (NC > 0)
                    streams_product_wt<NC, 2>(acc[0], s_X, 2 * kATileBytes, kATileBytes, ro, s_w + warp_uniform(P.g.w_hi[l]), s_w + warp_uniform(P.g.w_lo[l]), warp_uniform(P.g.Kp[l]), warp_uniform(P.g.Np[l]), n0);
                if (dw) issue_dw16(dwa, s_X, s_Y, 16 * wgi, !first_tile);
                umma::wgmma_commit();
                umma::wgmma_wait0();
            };
            if (nn == 32) products(std::integral_constant<int, 32>());
            else if (nn == 16) products(std::integral_constant<int, 16>());
            else products(std::integral_constant<int, 0>());
            if (dw) {
#pragma unroll
                for (int q = 0; q < 2; q++) dws[q * kBwdThreads] = make_float4(dwa[4 * q], dwa[4 * q + 1], dwa[4 * q + 2], dwa[4 * q + 3]);
            }
            __syncthreads();                                   // every product of this step has read X and Y
            if (l == 1 && tid == 0) {          // Y is free: bring a_0 | ta_0 back for the last step
                umma::mbar_expect_tx(&bars[0], (uint32_t)kSetBytes);
                umma::bulk_g2s(s_Y, out.a0_spill + (size_t)tile * kSetBytes, (uint32_t)kSetBytes, &bars[0]);
            }
            if (l == 0 && tid == 0 && tile + (int)gridDim.x < ntiles) {     // X is free: the next tile's a_0 | ta_0
                umma::mbar_expect_tx(&bars[1], (uint32_t)kSetBytes);
                umma::bulk_g2s(s_X, out.a0_spill + (size_t)(tile + gridDim.x) * kSetBytes, (uint32_t)kSetBytes, &bars[1]);
            }
            if (l > 0) {
                if (nn > 0) {
                    // zbar_l = gelu'(z_l) abar_l + gelu''(z_l) tz_l tabar_l, tzbar_l = gelu'(z_l) tabar_l -> X; acc[0] keeps zbar_l of the
                    // valid rows (0 elsewhere) for the bias gradient of layer l - 1
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        if (8 * j < nn) {
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const int r = frag_row(mh, h), c = n0 + frag_col(j);
                                float zb[2], tzb[2];
#pragma unroll
                                for (int b = 0; b < 2; b++) {
                                    const int i = 4 * j + 2 * h + b;
                                    zb[b] = g1[i] * acc[0][i] + g2t[i] * acc[1][i];
                                    tzb[b] = g1[i] * acc[1][i];
                                }
                                store_pair(s_X, s_X + kATileBytes, r, c, zb[0], zb[1]);
                                store_pair(s_X + 2 * kATileBytes, s_X + 3 * kATileBytes, r, c, tzb[0], tzb[1]);
                                const bool rv = h ? rvalid1 : rvalid0;
                                acc[0][4 * j + 2 * h] = rv ? zb[0] : 0.f;
                                acc[0][4 * j + 2 * h + 1] = rv ? zb[1] : 0.f;
                            }
                        }
                    }
                    // bias gradient: column sums over each 32-row group (warps 2p, 2p + 1 of the warpgroup) in the order of the per-row
                    // colsum16 (frag_pair_colsum)
                    const int pair = 2 * wgi + ((warp & 3) >> 1);
                    float cs;
                    int col;
                    if (frag_pair_colsum(acc[0], nn, s_bx + pair * 16 * 32, 1 + pair, cs, col)) {
                        if (det) fx_add(&s_gb[(l - 1) * 64 + n0 + col], cs);
                        else atomicAdd(&s_gbf[(l - 1) * 64 + n0 + col], cs);
                    }
                }
                if (l >= 2) {
                    // a_{l-1} | ta_{l-1} -> Y and the GELU' / GELU'' factors of the next step from this thread's stashed z_{l-1} | tz_{l-1}
                    // (the forward layer l - 2 split its columns as the reverse step l - 1 does)
                    int m0, mn;
                    split_n(warp_uniform(P.g.Kp[l - 1]), nh, m0, mn);
                    float z[2][16];
#pragma unroll
                    for (int s = 0; s < 2; s++)
#pragma unroll
                        for (int j = 0; j < 4; j++) {
                            const float4 v = (8 * j < mn) ? stash[(8 * (l - 2) + 4 * s + j) * kBwdThreads] : make_float4(0.f, 0.f, 0.f, 0.f);
                            z[s][4 * j] = v.x; z[s][4 * j + 1] = v.y; z[s][4 * j + 2] = v.z; z[s][4 * j + 3] = v.w;
                        }
                    const float* bias = reinterpret_cast<const float*>(s_w + warp_uniform(P.g.bias[l - 2]));
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        if (8 * j < mn) {
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const int r = frag_row(mh, h), c = m0 + frag_col(j);
                                float a[2], ta[2];
#pragma unroll
                                for (int b = 0; b < 2; b++) {
                                    const int i = 4 * j + 2 * h + b;
                                    activation(z[0][i], z[1][i], bias[c + b], a[b], ta[b], g1[i], g2t[i]);
                                }
                                store_pair(s_Y, s_Y + kATileBytes, r, c, a[0], a[1]);
                                store_pair(s_Y + 2 * kATileBytes, s_Y + 3 * kATileBytes, r, c, ta[0], ta[1]);
                            }
                        }
                    }
                }
            } else if (nn > 0) {
                // abar_0 | tabar_0 -> the exchange region, for k_sdf_lattice_scatter: a thread's column pair 8 j + 2 (t % 4) is one level
                float4* dst = out.xch + (size_t)tile * kTile;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int lv = (n0 + frag_col(j)) >> 1;
                    if (8 * j < nn && lv < P.L) {
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int i = 4 * j + 2 * h;
                            dst[(size_t)lv * out.xch_stride + frag_row(mh, h)] = make_float4(acc[0][i], acc[0][i + 1], acc[1][i], acc[1][i + 1]);
                        }
                    }
                }
            }
            PSDF_PHASE(kPhReverse3 + (3 - l));
        }
        ld_phase ^= 1;
        // no barrier before the next tile: X and Y were last read by this tile's step-0 products, complete before its second barrier
        // (the next tile's X arrives by TMA, behind the mbarrier); s_bx (= s_seed) was last read in step 1, before the step-0 barriers
        if (out.phase_cycles && tid == 0) atomicAdd(out.phase_cycles + kPhTiles, 1ull);
    }
    // ---------------- weight gradients of this CTA: this thread's stashed dW fragments -> the CTA's slab (plain stores; k_dw_reduce adds
    // up the CTAs' slabs). Element 4 j + 2 h + b of dW_l is row 16 (warp & 3) + lane / 4 + 8 h, column 16 wgi + 8 j + 2 (lane % 4) + b; the
    // thread's columns past K_l (up to Kp_l) are written too and never read
    if (!first_tile) {
        unsigned long long* dw = g_dw_sdf_bwd + (size_t)blockIdx.x * kDwSlots;          // deterministic mode
        float* dwf = reinterpret_cast<float*>(g_dw_sdf_bwd) + (size_t)blockIdx.x * kDwSlots;   // float mode
#pragma unroll 1
        for (int l = 0; l < kNL; l++) {
            if (16 * wgi >= P.g.Kp[l]) continue;
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const float4 v = stash[(kStashDw + 2 * l + j) * kBwdThreads];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int m = 16 * (warp & 3) + lane / 4 + 8 * h, k = 16 * wgi + 8 * j + 2 * (lane & 3);
                    const float v0 = h ? v.z : v.x, v1 = h ? v.w : v.y;
                    const int slot = l * kDwLd * kDwLd + m * kDwLd + k;
                    if (det) *reinterpret_cast<ulonglong2*>(dw + slot) = make_ulonglong2(fx_of(v0), fx_of(v1));
                    else *reinterpret_cast<float2*>(dwf + slot) = make_float2(v0, v1);
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

// workspace per 128-sample tile: the layer-0 operand tiles (a_0 | ta_0, 64 KB), written by k_sdf_input_tiles and read by TMA into the
// persistent kernel twice (forward recompute and the first layer's weight gradient), and the exchange rows abar_0 | tabar_0 (16 bytes per sample and level,
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
    for (int l = 0; l < kNL; l++) out.gbias[l] = gb[l];
    out.fx_mlp = dbuf ? dbuf->sdf_mlp : nullptr;
    uint8_t* a0_spill = workspace;
    out.a0_spill = a0_spill;
    out.xch = reinterpret_cast<float4*>(workspace + (size_t)tiles * kSetBytes);
    out.xch_stride = tiles * kTile;
    // diagnostics: PSDF_PHASE_TIMING=1 prints thread 0's clock64 breakdown per phase (average cycles per tile) after every launch
    static const bool timing = getenv("PSDF_PHASE_TIMING") && atoi(getenv("PSDF_PHASE_TIMING")) != 0;
    static unsigned long long* d_cycles = nullptr;
    static cudaEvent_t ev[5];
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
    // the last region holds the upstream geometric-feature rows of a tile or, in the reverse sweep, the 8 x 16 x 32 fragments exchanged
    // for the bias column sums
    const size_t seed_bytes = std::max((size_t)kTile * (size_t)((out_dim - 1) | 1) * sizeof(float), (size_t)(8 * 16 * 32 * sizeof(float)));
    const size_t smem = (size_t)P.g.total + 2 * kSetBytes + kNL * 64 * sizeof(unsigned long long) + 64 + seed_bytes;
    if (smem > 227 * 1024) return PSDF_ERR_UNSUPPORTED;
    const long long tile_threads = (long long)tiles * (P.g.Kp[0] / 8) * kTile;
    k_sdf_input_tiles<D><<<(unsigned)div_up(tile_threads, (long long)kInputTileThreads), kInputTileThreads, 0, ST>>>(
        P, S, reinterpret_cast<const float2*>(lattice), scale_factor, shift, window, a0_spill);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[1], ST);
    { static bool optin_[64]; psdf::psdf_optin_smem(k_sdf_fused_backward<D>, 227 * 1024, optin_); }
    const int ctas = min(min(tiles, sms), kAccCtas);
    k_sdf_fused_backward<D><<<ctas, kBwdThreads, smem, ST>>>(P, S, blob, out);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[2], ST);
    {
        DwSums ds;
        for (int l = 0; l < kNL; l++) ds.gW[l] = gW[l];
        ds.fx_mlp = out.fx_mlp;
        ds.fx_w = kFxW;
        int max_nk = 0;
        for (int l = 0; l < kNL; l++) max_nk = max(max_nk, P.g.N[l] * P.g.K[l]);
        const dim3 grid(div_up(max_nk, kDwReduceThreads), kNL, kDwReduceChunks);
        if (dbuf) k_dw_reduce<kDwLd, unsigned long long, SdfDwSlab><<<grid, kDwReduceThreads, 0, ST>>>(P.g, ctas, ds);
        else k_dw_reduce<kDwLd, float, SdfDwSlab><<<grid, kDwReduceThreads, 0, ST>>>(P.g, ctas, ds);
        PSDF_CHECK_LAUNCH();
    }
    if (timing) cudaEventRecord(ev[3], ST);
    k_sdf_lattice_scatter<D><<<dim3(div_up(out.xch_stride, kScatterThreads), L), kScatterThreads, 0, ST>>>(
        P, S, out.xch, out.xch_stride, scale_factor, shift, window, grad_lattice, dbuf ? dbuf->sdf_lattice : nullptr);
    PSDF_CHECK_LAUNCH();
    if (timing) cudaEventRecord(ev[4], ST);
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
        float ms[4] = {0.f, 0.f, 0.f, 0.f};
        for (int i = 0; i < 4; i++) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
        fprintf(stderr, "[psdf_sdf_fused_backward N=%d tiles=%llu] cycles/tile: tile load wait %.0f forward %.0f seed %.0f rev3 %.0f rev2 %.0f rev1 %.0f "
                        "rev0 %.0f | flush/CTA %.0f | input tiles %.3f ms, fused kernel %.3f ms, weight-gradient reduction %.3f ms, lattice "
                        "scatter %.3f ms\n", total, h[kPhTiles], h[0] / t, h[1] / t, h[2] / t, h[3] / t, h[4] / t, h[5] / t, h[6] / t,
                (double)h[kPhFlush] / ctas, ms[0], ms[1], ms[2], ms[3]);
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
