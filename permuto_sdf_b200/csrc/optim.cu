// Dense fused AdamW sweep for the hash tables and MLP parameters (sm_90a).
// One pass over {param, grad, exp_avg, exp_avg_sq}: 28 B/parameter (read 16, write 12), optional gradient
// zeroing folded in (+4 B) so that no separate zero_grad memset is needed. Math = torch.optim.AdamW /
// apex FusedAdam as used by the reference (train_permuto_sdf.py:293-304: betas (0.9, 0.99), eps 1e-15,
// decoupled weight decay, no amsgrad):
//   p  <- p (1 - lr wd);  m <- b1 m + (1-b1) g;  v <- b2 v + (1-b2) g^2
//   p  <- p - lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// HBM-bound streaming kernel: 128-bit loads/stores, grid = multiple of the SM count, grid-stride loop.
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
__global__ void __launch_bounds__(256)
k_adamw(long long n, float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, float lr,
        float beta1, float beta2, float eps, float weight_decay, float bias_c1, float bias_c2_sqrt, const int* __restrict__ step_dev,
        const float* __restrict__ hyper_dev, float grad_scale, int zero_grad) {
    const long long n4 = n >> 2;
    if (hyper_dev) { lr = hyper_dev[0]; weight_decay = hyper_dev[1]; }   // schedule values kept in device memory (CUDA-graph replay)
    if (step_dev) {   // step count kept in device memory (CUDA-graph replay): bias corrections computed here
        const float t = (float)step_dev[0];
        bias_c1 = 1.0f - powf(beta1, t);
        bias_c2_sqrt = sqrtf(1.0f - powf(beta2, t));
    }
    const float decay = 1.0f - lr * weight_decay;
    const float step_size = lr / bias_c1;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // two independent float4 quadruples per thread and iteration: 8 x 16-byte loads in flight before the first use
    for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += 2 * stride) {
        const long long i1 = i0 + stride;
        const bool two = i1 < n4;
        float4 P[2], G[2], M[2], V[2];
        P[0] = reinterpret_cast<float4*>(p)[i0]; G[0] = reinterpret_cast<float4*>(g)[i0];
        M[0] = reinterpret_cast<float4*>(m)[i0]; V[0] = reinterpret_cast<float4*>(v)[i0];
        if (two) {
            P[1] = reinterpret_cast<float4*>(p)[i1]; G[1] = reinterpret_cast<float4*>(g)[i1];
            M[1] = reinterpret_cast<float4*>(m)[i1]; V[1] = reinterpret_cast<float4*>(v)[i1];
        }
#pragma unroll
        for (int q = 0; q < 2; q++) {
            if (q == 1 && !two) break;
            float* pp = &P[q].x; float* gg = &G[q].x; float* mm = &M[q].x; float* vv = &V[q].x;
#pragma unroll
            for (int k = 0; k < 4; k++) adamw_update(pp[k], mm[k], vv[k], gg[k], grad_scale, decay, step_size, beta1, beta2, bias_c2_sqrt, eps);
            const long long i = q ? i1 : i0;
            reinterpret_cast<float4*>(p)[i] = P[q];
            reinterpret_cast<float4*>(m)[i] = M[q];
            reinterpret_cast<float4*>(v)[i] = V[q];
            if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    // tail
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        long long i = (n4 << 2) + threadIdx.x;
        float pk = p[i], mk = m[i], vk = v[i];
        adamw_update(pk, mk, vk, g[i], grad_scale, decay, step_size, beta1, beta2, bias_c2_sqrt, eps);
        p[i] = pk; m[i] = mk; v[i] = vk;
        if (zero_grad) g[i] = 0.f;
    }
}
// ------------------------------------------------------------------------------------------------ data-parallel fused step
// One kernel = gradient reduction + AdamW + parameter broadcast over NVLink peer memory (no NCCL all-reduce, no second pass):
// rank r owns the shard [lo, hi) of every parameter group. For each element of its shard it
//   * loads the gradient from ALL ranks' gradient buffers (its own from HBM, the others through peer loads over NVLink / NVSwitch),
//   * sums them (grad_scale = 1 / world makes it the mean), updates ITS exp_avg / exp_avg_sq (optimizer state is sharded: only the
//     owner keeps it current) and the parameter,
//   * stores the new parameter into ALL ranks' parameter buffers (peer stores).
// Per rank and step: (W-1)/W of the gradient bytes in, (W-1)/W of the parameter bytes out, both directions at once, overlapped
// element by element with the optimizer arithmetic -- against all-reduce (2 (W-1)/W bytes each way) followed by a full local AdamW
// pass. The caller brackets the launch with a cross-rank barrier on each side (gradients final before, parameters landed after) and
// zeroes its own gradient buffer afterwards. Buffers live in CUDA peer-mapped (symmetric) memory.
struct PeerPtrs { float* p[8]; };
// NVSwitch multicast (NVLS): one multimem.ld_reduce returns the SUM of the word over every rank's buffer (the switch reduces), one
// multimem.st writes every rank's buffer (the switch replicates) -- inbound and outbound bytes per rank drop from (W-1)/W to 1/W of
// the buffer. Addresses are offsets into the multicast mapping of the symmetric allocation.
__device__ __forceinline__ float4 mc_ld_reduce(const float* mc) {
    float4 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
    return r;
}
__device__ __forceinline__ void mc_st(float* mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
template <int W, bool MC>
__global__ void __launch_bounds__(256)
k_adamw_dp(long long n, int rank, PeerPtrs grads, PeerPtrs params, float* __restrict__ mc_grad, float* __restrict__ mc_param,
           float* __restrict__ m, float* __restrict__ v, float lr, float beta1, float beta2, float eps, float weight_decay, float bias_c1,
           float bias_c2_sqrt, const int* __restrict__ step_dev, const float* __restrict__ hyper_dev, float grad_scale) {
    if (hyper_dev) { lr = hyper_dev[0]; weight_decay = hyper_dev[1]; }
    if (step_dev) {
        const float t = (float)step_dev[0];
        bias_c1 = 1.0f - powf(beta1, t);
        bias_c2_sqrt = sqrtf(1.0f - powf(beta2, t));
    }
    const float decay = 1.0f - lr * weight_decay;
    const float step_size = lr / bias_c1;
    const long long n4 = n >> 2;                         // the shard is a whole number of float4 (caller aligns)
    const long long stride = (long long)gridDim.x * blockDim.x;
    constexpr int U = 2;                                 // float4 per thread and iteration: U * W peer loads in flight before the first use
    for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += U * stride) {
        float4 G[U], P[U], M[U], V[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long i = i0 + u * stride;
            ok[u] = i < n4;
            G[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!ok[u]) continue;
            if (MC) G[u] = mc_ld_reduce(mc_grad + 4 * i);
            else {
                float4 g[W];
#pragma unroll
                for (int r = 0; r < W; r++) g[r] = __ldcg(reinterpret_cast<const float4*>(grads.p[(rank + r) % W]) + i);   // local copy first
#pragma unroll
                for (int r = 0; r < W; r++) { G[u].x += g[r].x; G[u].y += g[r].y; G[u].z += g[r].z; G[u].w += g[r].w; }
            }
            P[u] = reinterpret_cast<const float4*>(params.p[rank])[i];
            M[u] = reinterpret_cast<float4*>(m)[i];
            V[u] = reinterpret_cast<float4*>(v)[i];
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (!ok[u]) continue;
            const long long i = i0 + u * stride;
            float* pp = &P[u].x; float* gg = &G[u].x; float* mm = &M[u].x; float* vv = &V[u].x;
#pragma unroll
            for (int k = 0; k < 4; k++) adamw_update(pp[k], mm[k], vv[k], gg[k], grad_scale, decay, step_size, beta1, beta2, bias_c2_sqrt, eps);
            reinterpret_cast<float4*>(m)[i] = M[u];
            reinterpret_cast<float4*>(v)[i] = V[u];
            if (MC) mc_st(mc_param + 4 * i, P[u]);
            else {
#pragma unroll
                for (int r = 0; r < W; r++) reinterpret_cast<float4*>(params.p[(rank + r) % W])[i] = P[u];
            }
        }
    }
}
#define ST ((cudaStream_t)stream)
}  // namespace

// ---------------------------------------------------------------------------------------------- deterministic mode (common.cuh)
static psdf::DetBufs g_det[64];
static bool g_det_on[64];
namespace psdf {
const DetBufs* det_buffers() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < 64 && g_det_on[dev]) ? &g_det[dev] : nullptr;
}
}  // namespace psdf

extern "C" {
// Switch the training path's gradient reductions (and random occupancy updates) of the current device between float atomics (on = 0,
// the default) and the order-independent fixed-point sums of common.cuh (on = 1), whose results are the same in every run.
// lattice_entries = the largest L * T * F of a backward call, voxels = the largest occupancy grid. Allocates / frees device memory:
// call it outside CUDA-graph capture, with no launch of this library in flight.
int psdf_set_deterministic(int on, long long lattice_entries, long long voxels) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || lattice_entries < 0 || voxels < 0) return PSDF_ERR_ARG;
    DetBufs& d = g_det[dev];
    if (g_det_on[dev]) {
        cudaFree(d.sdf_lattice); cudaFree(d.sdf_mlp); cudaFree(d.rgb_lattice); cudaFree(d.rgb_mlp); cudaFree(d.neus); cudaFree(d.lip);
        cudaFree(d.loss); cudaFree(d.winner);
        g_det_on[dev] = false;
    }
    if (!on) return PSDF_OK;
    typedef unsigned long long U;
    const long long n_sdf = 4LL * kDetSdfW + 4 * 64, n_rgb = 4LL * kDetRgbW + 4 * 128, n_neus = 6LL * kDetImages + 1;
    const long long lat = lattice_entries > 0 ? lattice_entries : 1, vox = voxels > 0 ? voxels : 1;
    bool ok = cudaMalloc(&d.sdf_lattice, lat * sizeof(U)) == cudaSuccess && cudaMalloc(&d.rgb_lattice, lat * sizeof(U)) == cudaSuccess &&
              cudaMalloc(&d.sdf_mlp, n_sdf * sizeof(U)) == cudaSuccess && cudaMalloc(&d.rgb_mlp, n_rgb * sizeof(U)) == cudaSuccess &&
              cudaMalloc(&d.neus, n_neus * sizeof(U)) == cudaSuccess && cudaMalloc(&d.lip, 4 * sizeof(U)) == cudaSuccess &&
              cudaMalloc(&d.loss, 14 * sizeof(U)) == cudaSuccess && cudaMalloc(&d.winner, vox * sizeof(int)) == cudaSuccess;
    ok = ok && cudaMemset(d.sdf_lattice, 0, lat * sizeof(U)) == cudaSuccess && cudaMemset(d.rgb_lattice, 0, lat * sizeof(U)) == cudaSuccess &&
         cudaMemset(d.sdf_mlp, 0, n_sdf * sizeof(U)) == cudaSuccess && cudaMemset(d.rgb_mlp, 0, n_rgb * sizeof(U)) == cudaSuccess &&
         cudaMemset(d.neus, 0, n_neus * sizeof(U)) == cudaSuccess && cudaMemset(d.lip, 0, 4 * sizeof(U)) == cudaSuccess &&
         cudaMemset(d.loss, 0, 14 * sizeof(U)) == cudaSuccess && cudaMemset(d.winner, 0, vox * sizeof(int)) == cudaSuccess &&
         cudaDeviceSynchronize() == cudaSuccess;
    if (!ok) { cudaGetLastError(); return PSDF_ERR_LAUNCH; }
    d.lattice_len = lattice_entries; d.voxels = voxels;
    g_det_on[dev] = true;
    return PSDF_OK;
}
// step >= 1 is the (already incremented) step count, read from step_dev[0] instead when that is not NULL; pointers 16-byte aligned
int psdf_adamw_step(long long n, float* param, float* grad, float* exp_avg, float* exp_avg_sq, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int step, const int* step_dev, const float* hyper_dev, float grad_scale, int zero_grad,
                    void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    if (step < 1 && !step_dev) return PSDF_ERR_ARG;
    if (step < 1) step = 1;
    if ((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) != 0) return PSDF_ERR_ARG;
    double c1 = 1.0 - pow((double)beta1, (double)step);
    double c2 = 1.0 - pow((double)beta2, (double)step);
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    long long n4 = n >> 2;
    int blocks = (int)((n4 + 255) / 256);
    if (blocks < 1) blocks = 1;
    if (blocks > sms * 8) blocks = sms * 8;
    k_adamw<<<blocks, 256, 0, ST>>>(n, param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, (float)c1, (float)sqrt(c2),
                                   step_dev, hyper_dev, grad_scale, zero_grad);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// Data-parallel step of the shard [shard_lo, shard_lo + n) (elements, both multiples of 4) of one parameter group.
// grad_ptrs / param_ptrs: HOST arrays of `world` device pointers (entry r = the base of rank r's buffer for this group, peer-mapped
// into this process); exp_avg / exp_avg_sq: this rank's local moments of the group (full size, only the shard is touched).
int psdf_adamw_dp_step(long long n, long long shard_lo, int world, int rank, const uint64_t* grad_ptrs, const uint64_t* param_ptrs,
                       uint64_t mc_grad_ptr, uint64_t mc_param_ptr, float* exp_avg, float* exp_avg_sq, float lr, float beta1, float beta2,
                       float eps, float weight_decay, int step, const int* step_dev, const float* hyper_dev, float grad_scale, void* stream) {
    if (n < 0 || rank < 0 || rank >= world || (n & 3) || (shard_lo & 3) || !grad_ptrs || !param_ptrs) return PSDF_ERR_ARG;
    if (world != 1 && world != 2 && world != 4 && world != 8) return PSDF_ERR_UNSUPPORTED;
    if (n == 0) return PSDF_OK;
    if (step < 1 && !step_dev) return PSDF_ERR_ARG;
    if (step < 1) step = 1;
    PeerPtrs G, P;
    for (int r = 0; r < 8; r++) {
        G.p[r] = r < world ? reinterpret_cast<float*>((uintptr_t)grad_ptrs[r]) + shard_lo : nullptr;
        P.p[r] = r < world ? reinterpret_cast<float*>((uintptr_t)param_ptrs[r]) + shard_lo : nullptr;
        if (r < world && ((((uintptr_t)G.p[r]) | ((uintptr_t)P.p[r])) & 15)) return PSDF_ERR_ARG;
    }
    if ((((uintptr_t)(exp_avg + shard_lo)) | ((uintptr_t)(exp_avg_sq + shard_lo))) & 15) return PSDF_ERR_ARG;
    const bool mc = mc_grad_ptr != 0 && mc_param_ptr != 0;
    float* mcg = mc ? reinterpret_cast<float*>((uintptr_t)mc_grad_ptr) + shard_lo : nullptr;
    float* mcp = mc ? reinterpret_cast<float*>((uintptr_t)mc_param_ptr) + shard_lo : nullptr;
    const double c1 = 1.0 - pow((double)beta1, (double)step), c2 = 1.0 - pow((double)beta2, (double)step);
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long n4 = n >> 2;
    int blocks = (int)((n4 + 511) / 512);
    if (blocks < 1) blocks = 1;
    if (blocks > sms * 8) blocks = sms * 8;
#define PSDF_DP_LAUNCH(W, MC)                                                                                                        \
    k_adamw_dp<W, MC><<<blocks, 256, 0, ST>>>(n, rank, G, P, mcg, mcp, exp_avg + shard_lo, exp_avg_sq + shard_lo, lr, beta1, beta2, eps, \
                                              weight_decay, (float)c1, (float)sqrt(c2), step_dev, hyper_dev, grad_scale)
    if (mc) {
        if (world == 1) PSDF_DP_LAUNCH(1, true); else if (world == 2) PSDF_DP_LAUNCH(2, true);
        else if (world == 4) PSDF_DP_LAUNCH(4, true); else PSDF_DP_LAUNCH(8, true);
    } else {
        if (world == 1) PSDF_DP_LAUNCH(1, false); else if (world == 2) PSDF_DP_LAUNCH(2, false);
        else if (world == 4) PSDF_DP_LAUNCH(4, false); else PSDF_DP_LAUNCH(8, false);
    }
#undef PSDF_DP_LAUNCH
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
}  // extern "C"
