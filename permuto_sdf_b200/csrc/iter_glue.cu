// Glue of the direct (autograd-free) training iteration (train.py Trainer._iteration_direct), sm_90a. Each kernel replaces a chain of
// one-block PyTorch launches that the autograd formulation of train_permuto_sdf.py:311-422 spends between the big kernels:
//   k_iter_scalars      schedule ramps evaluated from the device-resident iteration number (map_range_val, common_utils.py:156-160) and
//                       inv_s = exp(10 * forced_variance) (SingleVarianceNetwork, volume_rendering_modules.py:94-114)             1 launch for ~12
//   k_lipschitz_pack    LipshitzMLP.normalization of the four colour-MLP matrices (models.py:96-110) + tensor-core operand packing   1 for 5
//   k_lipschitz_bwd4    its backward for the four layers, accumulated into the persistent .grad buffers (+ the Lipschitz-bound loss) 1 for 4 + 8
//   k_loss_terms        curvature values (models.py:283-294), all loss reductions (rgb L1, mask BCE, eikonal, curvature, off-surface
//                       exp(-100 |sdf|), Lipschitz bound), the weighted total and the off-surface gradient seed                      1 for ~30
//   k_sphere_fit_loss   sdf_loss_sphere of the sphere-fit phase (train_permuto_sdf.py:323-331): both reductions, the weighted total and
//                       the seeds d loss / d {sdf, grad}                                                                             1 for ~15
//   k_rand_points_u01   Sphere.rand_points_inside from one uniform draw [3,n]                                                          1 for 3
//   k_adamw_multi       AdamW over several parameter groups in one launch (optim.cu k_adamw per group otherwise)
#include <cstdlib>
#include "fused_rgb_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;
using namespace psdf_fused;

namespace {
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
#define ST ((cudaStream_t)stream)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    return v;
}
__device__ __forceinline__ float softplus_f(float x) { return x > 20.0f ? x : log1pf(expf(x)); }   // torch threshold 20
__device__ __forceinline__ float sigmoid_sp(float x) { return x > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-x)); }

// ---------------------------------------------------------------------------------------------- schedule scalars
struct Ramps {
    int n;
    float in0[8], in1[8], out0[8], scale[8];
    int kind[8];          // 0: ramp value, 1: exp(10 * ramp) (inv_s, unclipped), 2: exp(10 * ramp) clipped to [1e-6, 1e6]
};
__global__ void k_iter_scalars(Ramps R, const float* __restrict__ it_dev, float it_host, float* __restrict__ out) {
    const int i = threadIdx.x;
    if (i >= R.n) return;
    const float it = it_dev ? it_dev[0] : it_host;
    const float x = fminf(fmaxf(it, R.in0[i]), R.in1[i]);
    // same operation order (and roundings) as map_range_val on a float32 tensor: out0 + scale * (x - in0)
    float v = __fadd_rn(R.out0[i], __fmul_rn(R.scale[i], __fsub_rn(x, R.in0[i])));
    if (R.kind[i] >= 1) v = expf(__fmul_rn(v, 10.0f));
    if (R.kind[i] == 2) v = fminf(fmaxf(v, 1e-6f), 1e6f);
    out[i] = v;
}

// ---------------------------------------------------------------------------------------------- Lipschitz normalisation + packing
struct Lip4 {
    const float* W[kNL];
    const float* b[kNL];
    const float* c[kNL];
};
// one warp per padded output row n of layer blockIdx.y: scale = min(1, softplus(c) / sum|W[n,:]|), then W_eff -> bf16 hi/lo in the UMMA
// K-major core-matrix layout (and the transposed copy) exactly like fused_common.cuh k_pack_mlp
__global__ void __launch_bounds__(kThreads)
k_lipschitz_pack(MlpGeom g, Lip4 A, uint8_t* __restrict__ blob) {
    const int l = blockIdx.y;
    const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (n >= g.Np[l]) return;
    const int K = g.K[l], Kp = g.Kp[l];
    const bool real = n < g.N[l];
    const float* w = A.W[l] + (size_t)n * K;
    float a = 0.f;
    if (real) for (int j = lane; j < K; j += 32) a += fabsf(w[j]);
    a = warp_sum(a);
    const float s = real ? fminf(softplus_f(A.c[l][0]) / a, 1.0f) : 0.0f;
    const int sbo = (Kp / 8) * kLBO, sbo_t = (g.Np[l] / 8) * kLBO;
    for (int k = lane; k < Kp; k += 32) {
        const float v = (real && k < K) ? w[k] * s : 0.0f;
        __nv_bfloat16 hi, lo;
        umma::split_bf16(v, hi, lo);
        const int off = (n / 8) * sbo + (k / 8) * kLBO + (n % 8) * 16 + (k % 8) * 2;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.w_hi[l] + off) = hi;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.w_lo[l] + off) = lo;
        const int off_t = (k / 8) * sbo_t + (n / 8) * kLBO + (k % 8) * 16 + (n % 8) * 2;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.total + g.t_hi[l] + off_t) = hi;
        *reinterpret_cast<__nv_bfloat16*>(blob + g.total + g.t_lo[l] + off_t) = lo;
    }
    if (lane == 0) reinterpret_cast<float*>(blob + g.bias[l])[n] = real ? A.b[l][n] : 0.0f;
}

struct Lip4Bwd {
    unsigned long long* fx;          // deterministic mode: DetBufs::lip (d loss / d c_l in fixed point), else NULL
    const float* W[kNL];
    const float* c[kNL];
    float* G[kNL];        // d loss / d W_eff (read, then reset to zero for the next iteration)
    float* gW[kNL];       // (+=)
    float* gc[kNL];       // (+=)
    int rows[kNL], cols[kNL];
    float lip_weight;     // weight of the Lipschitz-bound loss prod_l softplus(c_l) (0: term inactive)
};
// rgb_misc.cu k_lipschitz_backward for all four layers in one launch, accumulating:
//   dW += G s - [ratio <= 1] sp / A^2 sign(W) D,   dc += [ratio <= 1] D / A sigmoid(c)   (D = sum_j G_j W_j)
// plus d (lip_weight prod_l softplus(c_l)) / d c_l
__global__ void __launch_bounds__(kThreads)
k_lipschitz_bwd4(Lip4Bwd A) {
    const int l = blockIdx.y;
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int rows = A.rows[l], cols = A.cols[l];
    if (r == 0 && lane == 0 && A.lip_weight != 0.0f) {
        float prod = A.lip_weight;
        for (int q = 0; q < kNL; q++) if (q != l) prod *= softplus_f(A.c[q][0]);
        if (A.fx) fx_add(A.fx + l, prod * sigmoid_sp(A.c[l][0]));
        else atomicAdd(A.gc[l], prod * sigmoid_sp(A.c[l][0]));
    }
    if (r >= rows) return;
    const float* W = A.W[l] + (size_t)r * cols;
    float* G = A.G[l] + (size_t)r * cols;
    float a = 0.f, d = 0.f;
    for (int j = lane; j < cols; j += 32) {
        const float w = W[j];
        a += fabsf(w);
        d += G[j] * w;
    }
    a = warp_sum(a);
    d = warp_sum(d);
    const float cv = A.c[l][0], sp = softplus_f(cv);
    const float ratio = sp / a;
    const bool active = ratio <= 1.0f;
    const float s = fminf(ratio, 1.0f);
    const float k = active ? sp / (a * a) * d : 0.0f;
    float* gW = A.gW[l] + (size_t)r * cols;
    for (int j = lane; j < cols; j += 32) {
        const float w = W[j];
        const float sg = w > 0.f ? 1.f : (w < 0.f ? -1.f : 0.f);
        gW[j] += G[j] * s - k * sg;
        G[j] = 0.0f;
    }
    if (lane == 0 && active) {
        if (A.fx) fx_add(A.fx + l, d / a * sigmoid_sp(cv));
        else atomicAdd(A.gc[l], d / a * sigmoid_sp(cv));
    }
}

// ---------------------------------------------------------------------------------------------- loss terms
struct LossArgs {
    unsigned long long* fx;          // deterministic mode: DetBufs::loss (the sums in fixed point), else NULL
    int N;                           // rows of the sample buffers
    const int* nr_valid_dev;         // [1] valid rows (static-capacity containers) or NULL (all N)
    const int* nr_mean_dev;          // [1] divisor of the per-sample means (data-parallel: mean per-rank count) or NULL (= valid rows)
    const float* g;                  // [N,3] d sdf/dx at the samples
    const float* gs;                 // [N,3] at the shifted samples, NULL: no curvature term
    int R;
    const float* ray_loss;           // [R,3] {rgb L1, mask BCE, eikonal} per ray
    int n_off;
    const float* sdf_off;            // [n_off] sdf at the off-surface points, NULL: no term
    float* g_off;                    // [n_off] d loss / d sdf_off (=)
    float c_rgb, c_mask, w_eik, w_curv, w_off, w_lip;
    const float* w_curv_dev;         // optional device multiplier of w_curv
    const float* lip_c[kNL];         // Lipschitz bound parameters (w_lip != 0)
    float* acc;                      // [8] accumulators + ticket (zero on entry, left zero)
    float* loss;                     // [1]
    float* terms;                    // [12]: sum rgb L1, sum BCE, sum eikonal, mean curvature, mean off-surface, lipschitz bound, valid rows,
                                     //       divisor of the per-sample means, loss_rgb, loss_eikonal
};
__global__ void __launch_bounds__(kThreads)
k_loss_terms(LossArgs A) {
    __shared__ float red[5][kThreads / 32];
    __shared__ bool last;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nv = A.nr_valid_dev ? min(max(A.nr_valid_dev[0], 0), A.N) : A.N;
    float v[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (A.gs && i < nv) {
        // curvature = acos(clamp(normalize(g) . normalize(gs), -1 + 1e-6, 1 - 1e-6)) / pi  (same roundings as rgb_misc.cu k_curv_forward)
        const float gx = A.g[3 * i], gy = A.g[3 * i + 1], gz = A.g[3 * i + 2];
        const float sx = A.gs[3 * i], sy = A.gs[3 * i + 1], sz = A.gs[3 * i + 2];
        const float na = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz))), 1e-12f);
        const float nb = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(sx, sx), __fmul_rn(sy, sy)), __fmul_rn(sz, sz))), 1e-12f);
        const float ax = __fdiv_rn(gx, na), ay = __fdiv_rn(gy, na), az = __fdiv_rn(gz, na);
        const float bx = __fdiv_rn(sx, nb), by = __fdiv_rn(sy, nb), bz = __fdiv_rn(sz, nb);
        const float dot = __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
        v[3] = acosf(fminf(fmaxf(dot, -1.0f + 1e-6f), 1.0f - 1e-6f)) * 0.3183098861837907f;
    }
    if (i < A.R) { v[0] = A.ray_loss[3 * i]; v[1] = A.ray_loss[3 * i + 1]; v[2] = A.ray_loss[3 * i + 2]; }
    if (A.sdf_off && i < A.n_off) {
        const float s = A.sdf_off[i];
        const float e = expf(-1e2f * fabsf(s));
        v[4] = e;
        const float sg = s > 0.f ? 1.f : (s < 0.f ? -1.f : 0.f);
        A.g_off[i] = A.w_off / (float)A.n_off * (-1e2f * sg) * e;
    }
#pragma unroll
    for (int q = 0; q < 5; q++) {
        const float s = warp_sum(v[q]);
        if (lane == 0) red[q][warp] = s;
    }
    __syncthreads();
    if (threadIdx.x < 5) {
        float s = 0.f;
        for (int w = 0; w < kThreads / 32; w++) s += red[threadIdx.x][w];
        if (s != 0.0f) {
            if (A.fx) fx_add(A.fx + threadIdx.x, s);
            else atomicAdd(A.acc + threadIdx.x, s);
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned t = atomicAdd(reinterpret_cast<unsigned*>(A.acc + 7), 1u);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!last || threadIdx.x != 0) return;
    __threadfence();
    float sums[5];
    if (A.fx) {
        volatile unsigned long long* fx = A.fx;
        for (int q = 0; q < 5; q++) { sums[q] = (float)((double)(long long)fx[q] / kFxScale); fx[q] = 0ull; }
    } else {
        volatile float* acc = A.acc;
        for (int q = 0; q < 5; q++) sums[q] = acc[q];
    }
    const float l1 = sums[0], bce = sums[1], eik = sums[2], curv = sums[3], off = sums[4];
    const int cnt = max(A.nr_mean_dev ? A.nr_mean_dev[0] : nv, 1);
    const float curv_mean = curv / (float)cnt;
    const float off_mean = A.sdf_off ? off / (float)A.n_off : 0.0f;
    float lip = 0.0f;
    if (A.w_lip != 0.0f) {
        lip = 1.0f;
        for (int q = 0; q < kNL; q++) lip *= softplus_f(A.lip_c[q][0]);
    }
    const float wc = A.w_curv * (A.w_curv_dev ? A.w_curv_dev[0] : 1.0f);
    float loss = l1 * A.c_rgb + bce * A.c_mask + eik * (A.w_eik / (float)cnt);
    if (A.gs) loss += curv_mean * wc;
    if (A.sdf_off) loss += off_mean * A.w_off;
    if (A.w_lip != 0.0f) loss += lip * A.w_lip;
    A.loss[0] = loss;
    A.terms[0] = l1; A.terms[1] = bce; A.terms[2] = eik; A.terms[3] = curv_mean; A.terms[4] = off_mean; A.terms[5] = lip; A.terms[6] = (float)nv;
    A.terms[7] = (float)cnt;
    A.terms[8] = l1 * A.c_rgb;                 // the reference's loss_rgb (mean over rays and channels)
    A.terms[9] = eik / (float)cnt;             // loss_eikonal (mean over the samples)
#pragma unroll
    for (int q = 0; q < 8; q++) A.acc[q] = 0.0f;      // ticket (acc[7], as bits) included: ready for the next launch
}

// ---------------------------------------------------------------------------------------------- sphere-fit loss
struct SphereFitArgs {
    unsigned long long* fx;          // deterministic mode: DetBufs::loss + 5 (the two sums in fixed point), else NULL
    int N;
    const float* pos;                // [N,3]
    const float* sdf;                // [N]
    const float* g;                  // [N,3] d sdf/dx
    float radius, cx, cy, cz, scale, w_sdf, w_eik;
    float* g_sdf;                    // [N]   d loss / d sdf (=)
    float* g_grad;                   // [N,3] d loss / d (d sdf/dx) (=)
    float* acc;                      // [4] accumulators + ticket (zero on entry, left zero)
    float* loss;                     // [1]
    float* terms;                    // [2]: loss_sdf, loss_eik
};
// sdf_loss_sphere (train.py, permuto_sdf_utils.py:53-77): w_sdf mean((sdf - (|p - c| - r) s)^2) + w_eik mean((|g| - s)^2), with the
// seeds of both terms written per row. |g| = 0 gives a zero eikonal seed (torch's norm backward at 0).
__global__ void __launch_bounds__(kThreads)
k_sphere_fit_loss(SphereFitArgs A) {
    __shared__ float red[2][kThreads / 32];
    __shared__ bool last;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float v[2] = {0.f, 0.f};
    if (i < A.N) {
        const float inv_n = 1.0f / (float)A.N;
        const float px = A.pos[3 * i] - A.cx, py = A.pos[3 * i + 1] - A.cy, pz = A.pos[3 * i + 2] - A.cz;
        const float d = (sqrtf(px * px + py * py + pz * pz) - A.radius) * A.scale;
        const float e = A.sdf[i] - d;
        v[0] = e * e;
        A.g_sdf[i] = 2.0f * A.w_sdf * e * inv_n;
        const float gx = A.g[3 * i], gy = A.g[3 * i + 1], gz = A.g[3 * i + 2];
        const float n = sqrtf(gx * gx + gy * gy + gz * gz);
        const float r = n - A.scale;
        v[1] = r * r;
        const float k = n > 0.0f ? 2.0f * A.w_eik * r / n * inv_n : 0.0f;
        A.g_grad[3 * i] = k * gx; A.g_grad[3 * i + 1] = k * gy; A.g_grad[3 * i + 2] = k * gz;
    }
#pragma unroll
    for (int q = 0; q < 2; q++) {
        const float s = warp_sum(v[q]);
        if (lane == 0) red[q][warp] = s;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        float s = 0.f;
        for (int w = 0; w < kThreads / 32; w++) s += red[threadIdx.x][w];
        if (s != 0.0f) {
            if (A.fx) fx_add(A.fx + threadIdx.x, s);
            else atomicAdd(A.acc + threadIdx.x, s);
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned t = atomicAdd(reinterpret_cast<unsigned*>(A.acc + 3), 1u);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!last || threadIdx.x != 0) return;
    __threadfence();
    float sums[2];
    if (A.fx) {
        volatile unsigned long long* fx = A.fx;
        for (int q = 0; q < 2; q++) { sums[q] = (float)((double)(long long)fx[q] / kFxScale); fx[q] = 0ull; }
    } else {
        volatile float* acc = A.acc;
        for (int q = 0; q < 2; q++) sums[q] = acc[q];
    }
    const float l_sdf = sums[0] / (float)A.N, l_eik = sums[1] / (float)A.N;
    A.loss[0] = l_sdf * A.w_sdf + l_eik * A.w_eik;
    A.terms[0] = l_sdf;
    A.terms[1] = l_eik;
#pragma unroll
    for (int q = 0; q < 4; q++) A.acc[q] = 0.0f;      // ticket (acc[3], as bits) included: ready for the next launch
}

// ---------------------------------------------------------------------------------------------- random points in a sphere
// src/Sphere.cu rand_points_inside: phi in [0, 2 pi), cos(theta) in [-1, 1), u in [0, 1) -> r = R u^(1/3) along the sphere direction
__global__ void k_rand_points_u01(int n, float radius, const float* __restrict__ u01 /* [3,n] */, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float phi = u01[i] * 6.283185307179586f;
    const float costheta = u01[n + i] * 2.0f - 1.0f;
    const float u = u01[2 * n + i];
    const float theta = acosf(costheta);
    const float r = radius * (float)pow((double)u, 1.0 / 3);          // same expressions as rayops.cu k_sphere_rand_points
    const float st = sinf(theta);
    out[3 * i] = r * st * cosf(phi);
    out[3 * i + 1] = r * st * sinf(phi);
    out[3 * i + 2] = r * cosf(theta);
}

// ---------------------------------------------------------------------------------------------- multi-group AdamW
struct AdamGroups {
    int n_groups;
    long long off4[9];            // prefix sums of the groups' float4 counts
    float* p[8]; float* g[8]; float* m[8]; float* v[8];
    const float* hyper_dev[8];    // [2] {lr, weight_decay} per group
};
template <int U>
__global__ void __launch_bounds__(256)
k_adamw_multi(AdamGroups A, float beta1, float beta2, float eps, const int* __restrict__ step_dev, int step_offset, float grad_scale) {
    // same arithmetic, in the same order, as optim.cu k_adamw (device-resident step count and hyper-parameters). U float4 quadruples
    // {p, g, m, v} per thread and iteration: 4 U 16-byte loads in flight before the first use, so that FEW resident blocks saturate HBM
    const float t = (float)(step_dev[0] + step_offset);
    const float bias_c1 = 1.0f - powf(beta1, t);
    const float bias_c2_sqrt = sqrtf(1.0f - powf(beta2, t));
    const long long total = A.off4[A.n_groups];
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += U * stride) {
        float4 P[U], G[U], M[U], V[U];
        long long j[U];
        int gi[U];
        bool ok[U];
#pragma unroll
        for (int q = 0; q < U; q++) {
            const long long i = i0 + q * stride;
            ok[q] = i < total;
            gi[q] = 0; j[q] = 0;
            if (!ok[q]) continue;
            int g = 0;
            while (g + 1 < A.n_groups && i >= A.off4[g + 1]) g++;
            gi[q] = g; j[q] = i - A.off4[g];
            P[q] = reinterpret_cast<float4*>(A.p[g])[j[q]]; G[q] = reinterpret_cast<float4*>(A.g[g])[j[q]];
            M[q] = reinterpret_cast<float4*>(A.m[g])[j[q]]; V[q] = reinterpret_cast<float4*>(A.v[g])[j[q]];
        }
#pragma unroll
        for (int q = 0; q < U; q++) {
            if (!ok[q]) continue;
            const float lr = A.hyper_dev[gi[q]][0], wd = A.hyper_dev[gi[q]][1];
            const float decay = 1.0f - lr * wd;
            const float step_size = lr / bias_c1;
            float* pp = &P[q].x; float* gg = &G[q].x; float* mm = &M[q].x; float* vv = &V[q].x;
#pragma unroll
            for (int k = 0; k < 4; k++) adamw_update(pp[k], mm[k], vv[k], gg[k], grad_scale, decay, step_size, beta1, beta2, bias_c2_sqrt, eps);
            reinterpret_cast<float4*>(A.p[gi[q]])[j[q]] = P[q];
            reinterpret_cast<float4*>(A.m[gi[q]])[j[q]] = M[q];
            reinterpret_cast<float4*>(A.v[gi[q]])[j[q]] = V[q];
            reinterpret_cast<float4*>(A.g[gi[q]])[j[q]] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}
}  // namespace

extern "C" {

// out[i] = ramp_i(iteration) = out0 + (out1 - out0) / (in1 - in0) * (clamp(iteration, in0, in1) - in0), kind 1 / 2: exp(10 * ramp)
// (unclipped / clipped to [1e-6, 1e6]). params [n,4] = {in0, in1, out0, out1} (host), kinds [n] (host); iteration from it_dev [1]
// (device float) or, when NULL, it_host. n <= 8.
int psdf_iter_scalars(int n, const float* params, const int* kinds, const float* it_dev, float it_host, float* out, void* stream) {
    if (n < 1 || n > 8 || !params || !kinds || !out) return PSDF_ERR_ARG;
    Ramps R;
    R.n = n;
    for (int i = 0; i < n; i++) {
        R.in0[i] = params[4 * i]; R.in1[i] = params[4 * i + 1]; R.out0[i] = params[4 * i + 2];
        // the Python expression (output_end - output_start) / (input_end - input_start) is evaluated in double and rounded when it
        // meets the float32 tensor
        R.scale[i] = (float)(((double)params[4 * i + 3] - (double)params[4 * i + 2]) / ((double)params[4 * i + 1] - (double)params[4 * i]));
        R.kind[i] = kinds[i];
    }
    k_iter_scalars<<<1, 32, 0, ST>>>(R, it_dev, it_host, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// LipshitzMLP.normalization (models.py:96-110) of the four colour-MLP matrices W_l [N_l, K_l] with their bound parameters c_l [1] and
// psdf_rgb_mlp_pack of the result, in one launch: blob as psdf_rgb_mlp_blob_bytes / psdf_rgb_mlp_pack define it.
int psdf_lipschitz_pack4(int in_dim, int h1, int h2, int h3, int out_dim, const float* W0, const float* b0, const float* c0, const float* W1,
                         const float* b1, const float* c1, const float* W2, const float* b2, const float* c2, const float* W3, const float* b3,
                         const float* c3, uint8_t* blob, void* stream) {
    if (in_dim > 128 || h1 > 128 || h2 > 128 || h3 > 128 || out_dim > 16) return PSDF_ERR_UNSUPPORTED;
    int dims[kNL + 1] = {in_dim, h1, h2, h3, out_dim};
    MlpGeom g = make_geom_dims(dims);
    Lip4 A;
    A.W[0] = W0; A.W[1] = W1; A.W[2] = W2; A.W[3] = W3;
    A.b[0] = b0; A.b[1] = b1; A.b[2] = b2; A.b[3] = b3;
    A.c[0] = c0; A.c[1] = c1; A.c[2] = c2; A.c[3] = c3;
    dim3 grid(div_up(128 * 32, kThreads), kNL);
    k_lipschitz_pack<<<grid, kThreads, 0, ST>>>(g, A, blob);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// backward of the four normalisations in one launch: G_l = d loss / d W_eff_l [N_l, K_l] is consumed and RESET TO ZERO (it is the
// accumulation target of the next iteration's weight-gradient kernel), grad_W_l (+=), grad_c_l [1] (+=). lip_weight != 0 adds the
// gradient of lip_weight * prod_l softplus(c_l) (LipshitzMLP.lipshitz_bound_full, train_permuto_sdf.py:368-371).
int psdf_lipschitz_backward4(int in_dim, int h1, int h2, int h3, int out_dim, const float* W0, const float* c0, float* G0, float* gW0, float* gc0,
                             const float* W1, const float* c1, float* G1, float* gW1, float* gc1, const float* W2, const float* c2, float* G2,
                             float* gW2, float* gc2, const float* W3, const float* c3, float* G3, float* gW3, float* gc3, float lip_weight,
                             void* stream) {
    Lip4Bwd A;
    const DetBufs* dbuf = det_buffers();
    A.fx = dbuf ? dbuf->lip : nullptr;
    const int dims[kNL + 1] = {in_dim, h1, h2, h3, out_dim};
    A.W[0] = W0; A.W[1] = W1; A.W[2] = W2; A.W[3] = W3;
    A.c[0] = c0; A.c[1] = c1; A.c[2] = c2; A.c[3] = c3;
    A.G[0] = G0; A.G[1] = G1; A.G[2] = G2; A.G[3] = G3;
    A.gW[0] = gW0; A.gW[1] = gW1; A.gW[2] = gW2; A.gW[3] = gW3;
    A.gc[0] = gc0; A.gc[1] = gc1; A.gc[2] = gc2; A.gc[3] = gc3;
    int max_rows = 1;
    for (int l = 0; l < kNL; l++) { A.rows[l] = dims[l + 1]; A.cols[l] = dims[l]; max_rows = max(max_rows, dims[l + 1]); }
    A.lip_weight = lip_weight;
    dim3 grid(div_up(max_rows * 32, kThreads), kNL);
    k_lipschitz_bwd4<<<grid, kThreads, 0, ST>>>(A);
    PSDF_CHECK_LAUNCH();
    if (dbuf) {      // deterministic mode: fixed-point totals -> the float gradients (+=)
        FxSegs F;
        for (int l = 0; l < kNL; l++) F.add(dbuf->lip + l, A.gc[l], 1);
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    return PSDF_OK;
}

// All scalar loss terms of one training iteration (train_permuto_sdf.py:349-383) in one launch:
//   loss = c_rgb * sum_r L1_r + c_mask * sum_r BCE_r + w_eik * sum eik / n + w_curv * mean curvature + w_off * mean exp(-100 |sdf_off|)
//          + w_lip * prod softplus(c_l)
// with n = nr_mean_dev[0] (data-parallel runs: mean per-rank sample count) or the valid rows nr_valid_dev[0] (or N). grad / grad_shifted
// [N,3] (grad_shifted NULL: no curvature term), ray_loss [R,3] of psdf_neus_*_loss_forward, sdf_off [n_off] (NULL: no off-surface term)
// with its gradient seed g_off [n_off] = d loss / d sdf_off. acc [8]: scratch, ZERO before the first call, left zero by every call.
// terms [12] = {sum L1, sum BCE, sum eik, mean curvature, mean off-surface, Lipschitz bound, valid rows, n, loss_rgb, loss_eikonal, -, -}.
int psdf_loss_terms(int N, const int* nr_valid_dev, const int* nr_mean_dev, const float* grad, const float* grad_shifted, int R,
                    const float* ray_loss, int n_off, const float* sdf_off, float* g_off, float c_rgb, float c_mask, float w_eik, float w_curv,
                    const float* w_curv_dev, float w_off, float w_lip, const float* lip_c0, const float* lip_c1, const float* lip_c2,
                    const float* lip_c3, float* acc, float* loss, float* terms, void* stream) {
    if (N < 0 || R < 0 || n_off < 0 || !acc || !loss || !terms || (sdf_off && !g_off)) return PSDF_ERR_ARG;
    LossArgs A;
    const DetBufs* dbuf = det_buffers();
    A.fx = dbuf ? dbuf->loss : nullptr;
    A.N = N; A.nr_valid_dev = nr_valid_dev; A.nr_mean_dev = nr_mean_dev; A.g = grad; A.gs = grad_shifted; A.R = R; A.ray_loss = ray_loss;
    A.n_off = sdf_off ? n_off : 0; A.sdf_off = sdf_off; A.g_off = g_off;
    A.c_rgb = c_rgb; A.c_mask = c_mask; A.w_eik = w_eik; A.w_curv = w_curv; A.w_off = w_off; A.w_lip = w_lip; A.w_curv_dev = w_curv_dev;
    A.lip_c[0] = lip_c0; A.lip_c[1] = lip_c1; A.lip_c[2] = lip_c2; A.lip_c[3] = lip_c3;
    if (w_lip != 0.0f && (!lip_c0 || !lip_c1 || !lip_c2 || !lip_c3)) return PSDF_ERR_ARG;
    A.acc = acc; A.loss = loss; A.terms = terms;
    const int work = max(max(grad_shifted ? N : 0, R), max(A.n_off, 1));
    k_loss_terms<<<div_up(work, kThreads), kThreads, 0, ST>>>(A);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// Loss of one sphere-fit iteration (train_permuto_sdf.py:323-331) in one launch, see k_sphere_fit_loss. acc [4]: scratch, ZERO before the
// first call, left zero by every call. terms [2] = {loss_sdf, loss_eik} (unweighted means).
int psdf_sphere_fit_loss(int N, const float* pos, const float* sdf, const float* grad, float radius, const float center[3], float distance_scale,
                         float w_sdf, float w_eik, float* g_sdf, float* g_grad, float* acc, float* loss, float* terms, void* stream) {
    if (N < 1 || !pos || !sdf || !grad || !center || !g_sdf || !g_grad || !acc || !loss || !terms) return PSDF_ERR_ARG;
    SphereFitArgs A;
    const DetBufs* dbuf = det_buffers();
    A.fx = dbuf ? dbuf->loss + 5 : nullptr;
    A.N = N; A.pos = pos; A.sdf = sdf; A.g = grad;
    A.radius = radius; A.cx = center[0]; A.cy = center[1]; A.cz = center[2]; A.scale = distance_scale; A.w_sdf = w_sdf; A.w_eik = w_eik;
    A.g_sdf = g_sdf; A.g_grad = g_grad; A.acc = acc; A.loss = loss; A.terms = terms;
    k_sphere_fit_loss<<<div_up(N, kThreads), kThreads, 0, ST>>>(A);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// Sphere.rand_points_inside (src/Sphere.cu) from ONE uniform draw u01 [3,n] in [0,1): rows = phi / (2 pi), (cos(theta) + 1) / 2, u
int psdf_sphere_rand_points_inside_u01(int n, float radius, const float* u01, float* out, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_rand_points_u01<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, radius, u01, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// psdf_adamw_step over up to 8 parameter groups in one launch (device-resident step count and per-group {lr, weight_decay}; gradients
// are scaled by grad_scale and reset to zero). n_l % 4 == 0, pointers 16-byte aligned. The step is step_dev[0] + step_offset.
int psdf_adamw_multi_step(int n_groups, const long long* n, const uint64_t* param, const uint64_t* grad, const uint64_t* exp_avg,
                          const uint64_t* exp_avg_sq, const uint64_t* hyper_dev, float beta1, float beta2, float eps, const int* step_dev,
                          int step_offset, float grad_scale, int leave_room, void* stream) {
    if (n_groups < 1 || n_groups > 8 || !step_dev) return PSDF_ERR_ARG;
    AdamGroups A;
    A.n_groups = n_groups;
    long long off = 0;
    for (int i = 0; i < n_groups; i++) {
        if (n[i] % 4 != 0 || !hyper_dev[i]) return PSDF_ERR_ARG;
        A.off4[i] = off;
        off += n[i] / 4;
        A.p[i] = reinterpret_cast<float*>(param[i]); A.g[i] = reinterpret_cast<float*>(grad[i]); A.m[i] = reinterpret_cast<float*>(exp_avg[i]);
        A.v[i] = reinterpret_cast<float*>(exp_avg_sq[i]); A.hyper_dev[i] = reinterpret_cast<const float*>(hyper_dev[i]);
    }
    A.off4[n_groups] = off;
    if (off == 0) return PSDF_OK;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // Persistent grid-stride blocks. leave_room = 0: 8 blocks of 256 threads per SM, 2 float4 quadruples in flight per thread (the
    // fastest sweep on its own). leave_room != 0: 2 blocks per SM with 4 quadruples in flight -- most of the register file stays free, so
    // that the next iteration's ray generation / occupancy sampling kernels, replayed on another stream while this sweep runs
    // (Trainer._step_graphed), are co-resident instead of waiting for the sweep to drain. PSDF_ADAMW_BLOCKS_PER_SM / PSDF_ADAMW_UNROLL
    // override both for measurements.
    static const int per_sm_env = getenv("PSDF_ADAMW_BLOCKS_PER_SM") ? atoi(getenv("PSDF_ADAMW_BLOCKS_PER_SM")) : 0;
    static const int unroll_env = getenv("PSDF_ADAMW_UNROLL") ? atoi(getenv("PSDF_ADAMW_UNROLL")) : 0;
    const int per_sm = per_sm_env > 0 ? per_sm_env : (leave_room ? 2 : 8);
    const int unroll = unroll_env > 0 ? unroll_env : (leave_room ? 4 : 2);
    const long long blocks = (off + 255) / 256, cap = (long long)sms * per_sm;
    const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
    if (unroll >= 4) k_adamw_multi<4><<<grid, 256, 0, ST>>>(A, beta1, beta2, eps, step_dev, step_offset, grad_scale);
    else k_adamw_multi<2><<<grid, 256, 0, ST>>>(A, beta1, beta2, eps, step_dev, step_offset, grad_scale);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
