// Fused colour network for sm_90a: positions, view directions, sdf gradients and geometric features in -> linear RGB out
// (before colour calibration / sigmoid), i.e. RGB.forward of the reference (permuto_sdf_py/models/models.py:309-420):
//     feat = permutohedral_encoding(points) (+ concat points)        2L + 4 columns
//     x    = [feat | SH_5(view dir) (25) | normalize(sdf gradient) (3) | geom feature (32)]
//     y    = LipshitzMLP(x): K0 -> 128 -> 128 -> 64 -> 3, GELU between layers (weights already row-normalised by the caller)
// One CTA = one 128-sample tile = MMA M. Input columns are built in registers and written as bf16 hi/lo operand tiles
// ([128 x <=128] K-major core-matrix layout, 8-row-group stride 2048 B); every layer is three split products of
// wgmma (M64 x N<=64 x K16, the four warpgroups take one row half x column half each); the epilogue (bias + GELU) writes the next layer's tiles
// in place. Weights do not fit in shared memory next to the tiles, so each layer's hi/lo block streams in by one TMA bulk
// copy into a single buffer; the copy of layer l+1 is issued the moment layer l's MMAs retire and hides behind the epilogue.
// The backward pass (fused_rgb_bwd.cu) recomputes this forward, so nothing is saved for it.
#include "fused_common.cuh"
#include "fused_rgb_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;
using namespace psdf_rgb;

namespace {
__device__ float g_acc_rgb[(size_t)kAccCtas * kTile * 128];     // accumulator areas (umma.cuh)

__global__ void __launch_bounds__(kRgbThreads, 1)
k_rgb_fused(RgbParams P, const float* __restrict__ pos, const float* __restrict__ dirs, const float* __restrict__ sdf_grad,
            const float* __restrict__ geom, const float2* __restrict__ lattice, const float* __restrict__ scale,
            const float* __restrict__ shift, const float* __restrict__ window, const uint8_t* __restrict__ blob, float* __restrict__ out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_a = smem;                                   // operand tiles [hi | lo], 32 KB each
    uint8_t* s_w = s_a + 2 * kWTileBytes;                  // weights of the current layer [hi | lo]
    LevelC* lc = reinterpret_cast<LevelC*>(s_w + 2 * kWTileBytes);
    float* s_bias = reinterpret_cast<float*>(lc + 1);      // 4 x 128
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_bias + kNL * 128);      // [0] weights

    const int tid = threadIdx.x, warp = tid >> 5;
    const int row = tid & 127, grp = tid >> 7;
    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_fence_init();
        umma::acc_attach(g_acc_rgb + (size_t)blockIdx.x * kTile * 128, 128);
    }
    load_level_consts(lc, P.L, scale, shift, window, tid, kRgbThreads);
    for (int i = tid; i < kNL * 128; i += kRgbThreads) {
        int l = i >> 7, c = i & 127;
        s_bias[i] = (c < P.g.Np[l]) ? reinterpret_cast<const float*>(blob + P.g.bias[l])[c] : 0.0f;
    }
    __syncthreads();
    const uint32_t tmem_base = 0;
    uint32_t w_phase = 0;

    const int ntiles = (P.N + kTile - 1) / kTile;
    // weights of layer 0 for the first tile
    if (tid == 0 && blockIdx.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int n = tile * kTile + row;
        const bool valid = n < P.N;
        build_input_tile(P, lc, lattice, pos, dirs, sdf_grad, geom, n, valid, row, grp, s_a, s_a + kWTileBytes);
#pragma unroll 1
        for (int l = 0; l < kNL; l++) {
            umma::mbar_wait(&bars[0], w_phase);
            w_phase ^= 1;
            umma::fence_async_smem();
            __syncthreads();
            issue_gemm_w(tmem_base, warp >> 2, s_a, s_a + kWTileBytes, s_w, s_w + P.g.Np[l] * P.g.Kp[l] * 2, P.g.Kp[l], P.g.Np[l]);
            __syncthreads();
            // the weight buffer is free again: stream the next layer (or layer 0 of this CTA's next tile) behind the epilogue
            if (tid == 0) {
                if (l + 1 < kNL) load_layer_weights(s_w, blob, P.g, l + 1, false, &bars[0]);
                else if (tile + (int)gridDim.x < ntiles) load_layer_weights(s_w, blob, P.g, 0, false, &bars[0]);
            }
            const uint32_t trow = tmem_base + ((uint32_t)((warp & 3) * 32) << 16);
            if (l < kNL - 1) {
                for (int c = grp; c < P.g.Np[l] / 16; c += kRgbGroups) {
                    float z[16];
                    umma::tmem_ld16(trow + c * 16, z);
#pragma unroll
                    for (int i = 0; i < 16; i++) { const float zz = z[i] + s_bias[l * 128 + c * 16 + i]; z[i] = zz * gelu_eval(zz).cdf; }
                    store8w(s_a, s_a + kWTileBytes, row, 2 * c, z);
                    store8w(s_a, s_a + kWTileBytes, row, 2 * c + 1, z + 8);
                }
            } else if (grp == 0) {
                float z[16];
                umma::tmem_ld16(trow, z);
                if (valid) {
#pragma unroll
                    for (int i = 0; i < 3; i++) out[(size_t)n * 3 + i] = z[i] + s_bias[l * 128 + i];
                }
            }
        }
        __syncthreads();      // all accumulator reads / tile writes of this tile done before the next tile's encoder overwrites s_a
    }
}

#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {

long long psdf_rgb_mlp_blob_bytes(int in_dim, int h1, int h2, int h3, int out_dim) {
    int dims[kNL + 1] = {in_dim, h1, h2, h3, out_dim};
    MlpGeom g = make_geom_dims(dims);
    return (long long)g.total + g.total_t;
}

int psdf_rgb_mlp_pack(int in_dim, int h1, int h2, int h3, int out_dim, const float* W0, const float* b0, const float* W1, const float* b1,
                      const float* W2, const float* b2, const float* W3, const float* b3, uint8_t* blob, void* stream) {
    if (in_dim > 128 || h1 > 128 || h2 > 128 || h3 > 128 || out_dim > 16) return PSDF_ERR_UNSUPPORTED;
    int dims[kNL + 1] = {in_dim, h1, h2, h3, out_dim};
    MlpGeom g = make_geom_dims(dims);
    dim3 grid(div_up(128 * 128, 256), kNL);
    k_pack_mlp<<<grid, 256, 0, ST>>>(g, W0, b0, W1, b1, W2, b2, W3, b3, blob);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_rgb_fused_forward(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                           const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                           int h1, int h2, int h3, const uint8_t* blob, float* out, void* stream) {
    RgbParams P;
    int rc = make_rgb_params(P, N, L, T, geom_dim, points_scaling, h1, h2, h3);
    if (rc != PSDF_OK) return rc;
    if (N == 0) return PSDF_OK;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = (size_t)4 * kWTileBytes + sizeof(LevelC) + kNL * 128 * sizeof(float) + 64;
    { static bool optin_[64]; psdf::psdf_optin_smem(k_rgb_fused, 227 * 1024, optin_); }
    const int ntiles = div_up(N, kTile);
    k_rgb_fused<<<min(min(ntiles, sms), kAccCtas), kRgbThreads, smem, ST>>>(P, pos, dirs, sdf_grad, geom, reinterpret_cast<const float2*>(lattice),
                                                             scale_factor, shift, window, blob, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
