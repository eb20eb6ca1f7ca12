// Training backward of the fused colour network (sm_90a, wgmma): d loss / d (linear rgb) per sample in ->
// lattice gradient (scatter fused), d loss / d sdf-gradient (through the normalisation), d loss / d geom feature,
// weight + bias gradients of the 4 linear layers. Replaces loss.backward() through RGB.forward
// (permuto_sdf_py/models/models.py:395-414) -- encoding backward, 4 x (GELU backward, 2 GEMMs), normalize / cat backward.
//
// Per 128-sample tile (512 threads: row = tid & 127, group = tid >> 7):
//   1. input tile a_0 (encoder gather + SH + normal + geom) as in the forward; a_0 leaves by ONE TMA store (64 KB / tile, re-read from
//      L2 by the same CTA for dW_0: the only spill);
//   2. forward recompute, layers 0..2 on the tensor cores; pre-activations z^(0), z^(1), z^(2) STAY in the accumulator area
//      (128 + 128 + 64 columns);
//   3. reverse sweep l = 3..0: zbar^(l) tile -> MMA with W_l^T -> abar_l -> zbar^(l-1) = abar_l gelu'(z^(l-1)); beside that GEMM the
//      layer's input a_l is rebuilt from the stored z^(l-1) (a_0 returns by TMA) and the WEIGHT GRADIENT dW_l = zbar^(l)^T a_l is
//      formed on the tensor cores from the two tiles as they sit in shared memory: the sample axis is the MMA K dimension and an
//      operand tile in the K-major core-matrix layout is an MN-major operand for that product (see fused_sdf_bwd.cu). The issuing
//      warpgroups add the product from their registers to the CTA's fixed-point sums (each slot owned by one thread: no atomics); the
//      CTA flushes the four sums once, after its last tile -- 37 k reductions per CTA instead of per tile, with the same totals as a
//      per-tile fixed-point flush;
//      bias gradients = column sums (shuffles + shared atomics);
//   4. abar_0 -> lattice scatter (scatter_level without the tangent term: warp-aggregated red.global.add.v2.f32), normal -> sdf-gradient,
//      geom gradient.
// Deterministic mode (common.cuh): every gradient is summed in fixed point instead and added to the float gradients by the flush that
// follows the launch.
// Weights stream per layer through one 64 KB buffer by TMA; the next block is requested as soon as the MMAs that read the
// current one have retired, so the copy hides behind the epilogue.
// Accumulator map (umma.cuh): [0,128) z^(0) | [128,256) z^(1) | [256,384) z^(2) | [384,512) work. Weight-gradient sums: g_dw_rgb_bwd.
#include "fused_common.cuh"
#include "fused_rgb_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;
using namespace psdf_rgb;

namespace {
__device__ float g_acc_rgb_bwd[(size_t)kAccCtas * kTile * 512];     // accumulator areas (umma.cuh)
// weight-gradient sums of each CTA in fixed point (common.cuh fx_of), [CTA][layer][128 rows][128 columns]
constexpr int kDwSlots = kNL * 128 * 128;
__device__ unsigned long long g_dw_rgb_bwd[(size_t)kAccCtas * kDwSlots];
constexpr int kFxW = kDetRgbW, kFxB = 4 * kDetRgbW;    // weight / bias offsets in DetBufs::rgb_mlp
constexpr int kRgbSpillBytes = 2 * kWTileBytes;      // [hi | lo] of one operand tile

struct RgbSpill {
    uint8_t* a0;         // [ntiles][64 KB] input tiles a_0 (written and re-read by the same CTA)
    float* gW[kNL];      // [N_l, K_l] (+=)
    float* gbias[kNL];   // (+=)
    unsigned long long* fx_lattice;   // deterministic mode: fixed-point accumulators (DetBufs::rgb_lattice, ::rgb_mlp), else NULL
    unsigned long long* fx_mlp;
};
__global__ void __launch_bounds__(kRgbThreads, 1)
k_rgb_fused_backward(RgbParams P, const float* __restrict__ pos, const float* __restrict__ dirs, const float* __restrict__ sdf_grad,
                     const float* __restrict__ geom, const float2* __restrict__ lattice, const float* __restrict__ scale,
                     const float* __restrict__ shift, const float* __restrict__ window, const uint8_t* __restrict__ blob,
                     const float* __restrict__ g_out, float* __restrict__ grad_lattice, float* __restrict__ g_sdf_grad,
                     float* __restrict__ g_geom, RgbSpill sp) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_a = smem;                                   // activation tiles [hi | lo]
    uint8_t* s_z = s_a + 2 * kWTileBytes;                  // adjoint tiles [hi | lo]
    uint8_t* s_w = s_z + 2 * kWTileBytes;                  // weights of the current GEMM [hi | lo]
    LevelC* lc = reinterpret_cast<LevelC*>(s_w + 2 * kWTileBytes);
    float* s_bias = reinterpret_cast<float*>(lc + 1);      // 4 x 128
    // 4 x 128 bias-gradient accumulators of this CTA: float (s_gbf), or fixed point (s_gb) in deterministic mode
    unsigned long long* s_gb = reinterpret_cast<unsigned long long*>(s_bias + kNL * 128);
    float* s_gbf = reinterpret_cast<float*>(s_gb);
    const bool det = sp.fx_mlp != nullptr;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_gb + kNL * 128);   // [0] weights, [1] reverse MMAs, [2] dW MMAs, [3] a_0 reload
    // exchange tile abar_0: [128][K0 + 1] fp32 over s_a and, for K0 = 128 (L >= 28), the start of s_z; written after the last reverse
    // step's MMAs, the only readers of both, have completed
    float* s_x = reinterpret_cast<float*>(s_a);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row = tid & 127, grp = tid >> 7;
    const int K0 = P.g.Kp[0];
    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_init(&bars[1], 2 * 128);
        umma::mbar_init(&bars[2], 2 * 128);
        umma::mbar_init(&bars[3], 1);
        umma::mbar_fence_init();
        umma::acc_attach(g_acc_rgb_bwd + (size_t)blockIdx.x * kTile * 512, 512);
    }
    // reverse sweep: warpgroups 0 / 1 issue the row halves of the GEMM chain, warpgroups 2 / 3 the weight-gradient products beside it
    const int wgi = warp >> 2;
    const bool dw_issuer = wgi >= 2;
    load_level_consts(lc, P.L, scale, shift, window, tid, kRgbThreads);
    for (int i = tid; i < kNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        s_bias[i] = (c < P.g.Np[l]) ? reinterpret_cast<const float*>(blob + P.g.bias[l])[c] : 0.0f;
        s_gb[i] = 0ull;        // also clears s_gbf
    }
    __syncthreads();
    const uint32_t tmem_base = 0;
    const uint32_t tmem_z[3] = {tmem_base, tmem_base + 128, tmem_base + 256};
    const uint32_t tmem_work = tmem_base + 384;
    const uint32_t lane_off = (uint32_t)((warp & 3) * 32) << 16;
    uint32_t w_phase = 0, mma_phase = 0, dw_phase = 0, a0_phase = 0;
    unsigned long long* dw_cta = g_dw_rgb_bwd + (size_t)blockIdx.x * kDwSlots;    // this CTA's weight-gradient sums, layer l at l * 128 * 128

    const int ntiles = (P.N + kTile - 1) / kTile;
    if (tid == 0 && blockIdx.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const bool first_tile = tile == (int)blockIdx.x;
        const int n = tile * kTile + row;
        const bool valid = n < P.N;
        build_input_tile(P, lc, lattice, pos, dirs, sdf_grad, geom, n, valid, row, grp, s_a, s_a + kWTileBytes);

        // ---------------- forward recompute, layers 0..2
#pragma unroll 1
        for (int l = 0; l < 3; l++) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            if (l == 0 && tid == 0) {        // a_0 leaves as it is (needed again for dW_0 at the end of the reverse sweep)
                umma::bulk_s2g(sp.a0 + (size_t)tile * kRgbSpillBytes, s_a, kRgbSpillBytes);
                umma::bulk_commit();
            }
            issue_gemm_w(tmem_z[l], wgi, s_a, s_a + kWTileBytes, s_w, s_w + P.g.Np[l] * P.g.Kp[l] * 2, P.g.Kp[l], P.g.Np[l]);
            if (l == 0 && tid == 0) umma::bulk_wait_read0();      // s_a is overwritten by this layer's epilogue: the store must have read it
            __syncthreads();
            if (tid == 0) load_layer_weights(s_w, blob, P.g, l < 2 ? l + 1 : 3, l == 2, &bars[0]);   // W_{l+1}, then W_3^T
            for (int c = grp; c < P.g.Np[l] / 16; c += kRgbGroups) {
                float z[16];
                umma::tmem_ld16(tmem_z[l] + lane_off + c * 16, z);
#pragma unroll
                for (int i = 0; i < 16; i++) { const float zz = z[i] + s_bias[l * 128 + c * 16 + i]; z[i] = zz * gelu_eval(zz).cdf; }
                store8w(s_a, s_a + kWTileBytes, row, 2 * c, z);
                store8w(s_a, s_a + kWTileBytes, row, 2 * c + 1, z + 8);
            }
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
        // ---------------- reverse sweep, layers 3..0: s_z = zbar^(l), s_a = a_l (l = 3: still there from the forward)
#pragma unroll 1
        for (int l = 3; l >= 0; l--) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            const int Mdw = P.g.Np[l] > 64 ? 128 : 64;
            if (!dw_issuer) {
                // abar_l [128 x Kp_l] = zbar^(l) [128 x Np_l] W_l : B operand = W_l^T stored [Kp_l rows][Np_l]; both column halves
                for (int nh = 0; nh < 2; nh++)
                    issue_gemm_w(tmem_work, wgi + 2 * nh, s_z, s_z + kWTileBytes, s_w, s_w + P.g.Np[l] * P.g.Kp[l] * 2, P.g.Np[l], P.g.Kp[l]);
                umma::mbar_arrive(&bars[1]);
            }
            if (dw_issuer && l == 3) {                    // a_3 | zbar^(3) are both in place
                issue_dw_w(dw_cta + 3 * 128 * 128, wgi - 2, s_z, s_a, Mdw, P.g.Kp[3], first_tile);
                umma::mbar_arrive(&bars[2]);
            }
            // beside the MMAs: gelu'(z^(l-1)) of this thread's column chunks from the stored pre-activations, and the layer's
            // input a_l = gelu(z^(l-1)) back into s_a (its previous content a_(l+1) was last read by dW_(l+1), complete since the
            // previous step's epilogue waited for it)
            const int Kp = P.g.Kp[l];
            float g1a[16], g1b[16];                       // chunks grp and grp + 4 (Kp <= 128 -> at most two chunks per thread)
            if (l > 0) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int c = grp + j * kRgbGroups;
                    if (c < Kp / 16) {
                        float z[16];
                        umma::tmem_ld16(tmem_z[l - 1] + lane_off + c * 16, z);
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            const float zz = z[i] + s_bias[(l - 1) * 128 + c * 16 + i];
                            const GeluEval ge = gelu_eval(zz);
                            (j == 0 ? g1a : g1b)[i] = fmaf(zz, ge.pdf, ge.cdf);
                            z[i] = zz * ge.cdf;
                        }
                        if (l < 3) {
                            store8w(s_a, s_a + kWTileBytes, row, 2 * c, z);
                            store8w(s_a, s_a + kWTileBytes, row, 2 * c + 1, z + 8);
                        }
                    }
                }
            }
            if (l < 3) {
                if (l == 0 && tid == 0) {                 // a_0 returns by TMA (its store completed long ago)
                    umma::bulk_wait0();
                    umma::mbar_expect_tx(&bars[3], (uint32_t)kRgbSpillBytes);
                    umma::bulk_g2s(s_a, sp.a0 + (size_t)tile * kRgbSpillBytes, (uint32_t)kRgbSpillBytes, &bars[3]);
                }
                umma::fence_async_smem();
                __syncthreads();
                if (dw_issuer) {
                    if (l == 0) umma::mbar_wait(&bars[3], a0_phase);
                    issue_dw_w(dw_cta + l * 128 * 128, wgi - 2, s_z, s_a, Mdw, Kp, first_tile);
                    umma::mbar_arrive(&bars[2]);
                }
            }
            umma::mbar_wait(&bars[1], mma_phase);
            mma_phase ^= 1;
            if (tid == 0) {
                if (l > 0) load_layer_weights(s_w, blob, P.g, l - 1, true, &bars[0]);
                else if (tile + (int)gridDim.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
            }
            // s_z (and, for l = 0, the exchange tile over s_a) may only be written once the dW_l MMAs that read them have completed
            umma::mbar_wait(&bars[2], dw_phase);
            dw_phase ^= 1;
            if (l > 0) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int c = grp + j * kRgbGroups;
                    if (c >= Kp / 16) continue;
                    float ab[16];
                    umma::tmem_ld16(tmem_work + lane_off + c * 16, ab);
#pragma unroll
                    for (int i = 0; i < 16; i++) ab[i] *= (j == 0 ? g1a : g1b)[i];
                    store8w(s_z, s_z + kWTileBytes, row, 2 * c, ab);
                    store8w(s_z, s_z + kWTileBytes, row, 2 * c + 1, ab + 8);
                    if (!valid) {
#pragma unroll
                        for (int i = 0; i < 16; i++) ab[i] = 0.f;
                    }
                    int col;
                    const float cs = colsum16(ab, lane, col);
                    if (!(lane & 1)) {
                        if (det) fx_add(&s_gb[(l - 1) * 128 + c * 16 + col], cs);
                        else atomicAdd(&s_gbf[(l - 1) * 128 + c * 16 + col], cs);
                    }
                }
            } else {
                for (int c = grp; c < Kp / 16; c += kRgbGroups) {
                    float ab[16];
                    umma::tmem_ld16(tmem_work + lane_off + c * 16, ab);
#pragma unroll
                    for (int i = 0; i < 16; i++) s_x[row * (K0 + 1) + c * 16 + i] = ab[i];
                }
            }
        }
        a0_phase ^= 1;
        __syncthreads();
        // ---------------- encoder / tail backward from abar_0
        {
            const float* xr = s_x + row * (K0 + 1);
            float x[3] = {0.f, 0.f, 0.f};
            if (valid) { x[0] = pos[(size_t)n * 3]; x[1] = pos[(size_t)n * 3 + 1]; x[2] = pos[(size_t)n * 3 + 2]; }
            for (int l = grp; l < P.L; l += kRgbGroups) {
                const bool aggregate = lc->scale[l * 4] < kAggregateBelowScale;       // warp-uniform (l is)
                scatter_level<false>(x, nullptr, lc->scale + l * 4, lc->shift + l * 4, lc->window[l], xr[2 * l], xr[2 * l + 1], 0.f, 0.f, valid,
                                     aggregate, true, lane, P.cap_mask, (unsigned)P.T, grad_lattice + (size_t)l * P.T * 2,
                                     det ? sp.fx_lattice + (size_t)l * P.T * 2 : nullptr);
            }
            if (valid) {
                const int tail = P.enc_cols;          // SH at [tail, tail+25), normal at tail+25.., geom at tail+28..
                if (g_geom) {
                    float* gg = g_geom + (size_t)n * kGeomDim + grp * 8;
#pragma unroll
                    for (int i = 0; i < 8; i++) gg[i] = xr[tail + kShCols + 3 + grp * 8 + i];
                }
                if (grp == 3 && g_sdf_grad) {
                    const float gx = sdf_grad[(size_t)n * 3], gy = sdf_grad[(size_t)n * 3 + 1], gz = sdf_grad[(size_t)n * 3 + 2];
                    const float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
                    const float inv = 1.0f / fmaxf(nrm, 1e-12f);
                    const float bx = xr[tail + kShCols], by = xr[tail + kShCols + 1], bz = xr[tail + kShCols + 2];
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
        }
        __syncthreads();     // exchange tile / accumulators free for the next tile
    }
    __syncthreads();
    // ---- weight gradients of this CTA: fixed-point sums -> the deterministic accumulators (integer atomics, exact), or their float
    // value -> the gradients (+=)
    if ((int)blockIdx.x < ntiles) {
#pragma unroll 1
        for (int l = 0; l < kNL; l++) {
            const int K = P.g.K[l];
            const unsigned long long* src = dw_cta + l * 128 * 128;
            for (int i = tid; i < P.g.N[l] * K; i += kRgbThreads) {
                const int m = i / K, k = i - m * K;
                const unsigned long long v = src[m * 128 + k];
                if (v == 0ull) continue;
                if (det) atomicAdd(sp.fx_mlp + l * kFxW + i, v);
                else atomicAdd(sp.gW[l] + i, (float)((double)(long long)v / kFxScale));
            }
        }
    }
    for (int i = tid; i < kNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        if (det) { if (c < P.g.N[l] && s_gb[i] != 0ull) atomicAdd(sp.fx_mlp + kFxB + l * 128 + c, s_gb[i]); }
        else if (c < P.g.N[l] && s_gbf[i] != 0.0f) atomicAdd(sp.gbias[l] + c, s_gbf[i]);
    }
    if (tid == 0) umma::bulk_wait0();
}

#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {

// workspace: the input operand tiles a_0 (64 KB per 128-sample tile), written by TMA store in the forward recompute and read back by the
// same CTA for the first layer's weight gradient
long long psdf_rgb_fused_backward_workspace_bytes(int N) {
    const int ntiles = div_up(N > 0 ? N : 1, kTile);
    return (long long)ntiles * kRgbSpillBytes;
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
    static_assert((size_t)kTile * (128 + 1) * 4 <= (size_t)4 * kWTileBytes, "the exchange tile of K0 = 128 fits in s_a | s_z");
    const DetBufs* dbuf = det_buffers();
    if (dbuf && (long long)L * T * 2 > dbuf->lattice_len) return PSDF_ERR_UNSUPPORTED;   // reserve more with psdf_set_deterministic
    RgbSpill sp;
    float* b[kNL] = {gb0, gb1, gb2, gb3};
    float* w[kNL] = {gW0, gW1, gW2, gW3};
    for (int l = 0; l < kNL; l++) { sp.gbias[l] = b[l]; sp.gW[l] = w[l]; }
    sp.fx_lattice = dbuf ? dbuf->rgb_lattice : nullptr;
    sp.fx_mlp = dbuf ? dbuf->rgb_mlp : nullptr;
    sp.a0 = workspace;
    const int ntiles = div_up(N, kTile);
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = (size_t)6 * kWTileBytes + sizeof(LevelC) + kNL * 128 * (sizeof(float) + sizeof(unsigned long long)) + 64;
    // per device: set on every call (a second GPU needs its own opt-in)
    { static bool optin_[64]; psdf::psdf_optin_smem(k_rgb_fused_backward, 227 * 1024, optin_); }
    k_rgb_fused_backward<<<min(min(ntiles, sms), kAccCtas), kRgbThreads, smem, ST>>>(P, pos, dirs, sdf_grad, geom, reinterpret_cast<const float2*>(lattice),
                                                                      scale_factor, shift, window, blob, g_out, grad_lattice, g_sdf_grad, g_geom, sp);
    PSDF_CHECK_LAUNCH();
    if (dbuf) {      // deterministic mode: fixed-point totals -> the float gradients (+=)
        FxSegs F;
        F.add(dbuf->rgb_lattice, grad_lattice, (long long)L * T * 2);
        for (int l = 0; l < kNL; l++) {
            F.add(dbuf->rgb_mlp + l * kFxW, w[l], (long long)P.g.N[l] * P.g.K[l]);
            F.add(dbuf->rgb_mlp + kFxB + l * 128, b[l], P.g.N[l]);
        }
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
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
