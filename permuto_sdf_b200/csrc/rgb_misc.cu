// Small fused pieces around the colour network (sm_90a), each replacing a chain of tiny element-wise PyTorch launches:
//   * Lipschitz weight normalisation of LipshitzMLP (permuto_sdf_py/models/models.py:96-110):
//       W_eff[r,:] = W[r,:] * min(1, softplus(c) / sum_j |W[r,j]|)           forward + backward, one warp per row
//   * per-image colour calibration + sigmoid on packed samples (models.py:395-414, Colorcal :677-741):
//       rgb = sigmoid(x * (1 + weight_delta[img]) + bias[img]),  identity for img == idx_with_fixed_calib
//     forward + backward, one warp per ray (the per-image parameter gradients are reduced per ray, then one atomic per channel)
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr unsigned kFull = 0xffffffffu;
constexpr int kThreads = 256;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}
__device__ __forceinline__ float softplus_f(float x) { return x > 20.0f ? x : log1pf(expf(x)); }   // torch threshold 20

__global__ void __launch_bounds__(kThreads)
k_lipschitz_forward(int rows, int cols, const float* __restrict__ W, const float* __restrict__ c, float* __restrict__ W_eff) {
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (r >= rows) return;
    float a = 0.f;
    for (int j = lane; j < cols; j += 32) a += fabsf(W[(size_t)r * cols + j]);
    a = warp_sum(a);
    const float s = fminf(softplus_f(c[0]) / a, 1.0f);
    for (int j = lane; j < cols; j += 32) W_eff[(size_t)r * cols + j] = W[(size_t)r * cols + j] * s;
}
// dW = G s - [ratio <= 1] sp / A^2 sign(W) D,  dc += [ratio <= 1] D / A * sigmoid(c),  D = sum_j G_j W_j
__global__ void __launch_bounds__(kThreads)
k_lipschitz_backward(int rows, int cols, const float* __restrict__ W, const float* __restrict__ c, const float* __restrict__ G,
                     float* __restrict__ gW, float* __restrict__ gc) {
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (r >= rows) return;
    float a = 0.f, d = 0.f;
    for (int j = lane; j < cols; j += 32) {
        const float w = W[(size_t)r * cols + j];
        a += fabsf(w);
        d += G[(size_t)r * cols + j] * w;
    }
    a = warp_sum(a);
    d = warp_sum(d);
    const float cv = c[0], sp = softplus_f(cv);
    const float ratio = sp / a;
    const bool active = ratio <= 1.0f;               // torch.clamp(max=1) passes the gradient where ratio <= 1
    const float s = fminf(ratio, 1.0f);
    const float k = active ? sp / (a * a) * d : 0.0f;
    for (int j = lane; j < cols; j += 32) {
        const float w = W[(size_t)r * cols + j];
        const float sg = w > 0.f ? 1.f : (w < 0.f ? -1.f : 0.f);
        gW[(size_t)r * cols + j] = G[(size_t)r * cols + j] * s - k * sg;
    }
    if (lane == 0 && active && gc) {
        const float sig = cv > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-cv));
        atomicAdd(gc, d / a * sig);
    }
}

__global__ void __launch_bounds__(kThreads)
k_calib_sigmoid_forward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
                        const float* __restrict__ x, const int* __restrict__ img_idx, const float* __restrict__ weight_delta,
                        const float* __restrict__ bias, int fixed_img, float* __restrict__ out) {
    const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    RayRange rr = ray_range(ray, start_end, equal, fixed_n);
    if (rr.end > max_nr_samples || rr.n <= 0) return;
    float w[3] = {1.f, 1.f, 1.f}, b[3] = {0.f, 0.f, 0.f};
    if (img_idx) {
        const int im = img_idx[ray];
        if (im != fixed_img) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) { w[ch] = 1.0f + weight_delta[3 * im + ch]; b[ch] = bias[3 * im + ch]; }
        }
    }
    for (int e = lane; e < rr.n * 3; e += 32) {
        const int ch = e % 3;
        const size_t i = (size_t)rr.start * 3 + e;
        const float v = x[i] * w[ch] + b[ch];
        out[i] = 1.0f / (1.0f + expf(-v));
    }
}
__global__ void __launch_bounds__(kThreads)
k_calib_sigmoid_backward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
                         const float* __restrict__ x, const float* __restrict__ out, const float* __restrict__ g_out,
                         const int* __restrict__ img_idx, const float* __restrict__ weight_delta, int fixed_img, float* __restrict__ g_x,
                         float* __restrict__ g_weight_delta, float* __restrict__ g_bias) {
    const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    RayRange rr = ray_range(ray, start_end, equal, fixed_n);
    if (rr.end > max_nr_samples || rr.n <= 0) return;
    float w[3] = {1.f, 1.f, 1.f};
    int im = -1;
    if (img_idx) {
        im = img_idx[ray];
        if (im != fixed_img) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) w[ch] = 1.0f + weight_delta[3 * im + ch];
        } else im = -1;
    }
    float gw[3] = {0.f, 0.f, 0.f}, gb[3] = {0.f, 0.f, 0.f};
    // 96 = lcm(32, 3): within a 96-element chunk the channel of (q, lane) does not depend on the chunk
    for (int e0 = 0; e0 < rr.n * 3; e0 += 96) {
#pragma unroll
        for (int q = 0; q < 3; q++) {
            const int e = e0 + q * 32 + lane;
            if (e < rr.n * 3) {
                const int c = (q * 32 + lane) % 3;
                const size_t i = (size_t)rr.start * 3 + e;
                const float o = out[i];
                const float gv = g_out[i] * o * (1.0f - o);
                g_x[i] = gv * w[c];
                gw[c] += gv * x[i];
                gb[c] += gv;
            }
        }
    }
    if (im >= 0 && g_weight_delta) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float sw = warp_sum(gw[c]), sb = warp_sum(gb[c]);
            if (lane == 0) { atomicAdd(g_weight_delta + 3 * im + c, sw); atomicAdd(g_bias + 3 * im + c, sb); }
        }
    }
}
#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {
int psdf_lipschitz_normalize(int rows, int cols, const float* W, const float* c, float* W_eff, void* stream) {
    if (rows <= 0 || cols <= 0) return PSDF_ERR_ARG;
    k_lipschitz_forward<<<div_up((long long)rows * 32, kThreads), kThreads, 0, ST>>>(rows, cols, W, c, W_eff);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_lipschitz_normalize_backward(int rows, int cols, const float* W, const float* c, const float* grad_W_eff, float* grad_W,
                                      float* grad_c, void* stream) {
    if (rows <= 0 || cols <= 0) return PSDF_ERR_ARG;
    k_lipschitz_backward<<<div_up((long long)rows * 32, kThreads), kThreads, 0, ST>>>(rows, cols, W, c, grad_W_eff, grad_W, grad_c);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_calib_sigmoid_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x,
                               const int* img_idx, const float* weight_delta, const float* bias, int fixed_img, float* out,
                               void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_calib_sigmoid_forward<<<div_up((long long)nr_rays * 32, kThreads), kThreads, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, equal != 0,
                                                                                          fixed_n, x, img_idx, weight_delta, bias, fixed_img, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_calib_sigmoid_backward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* x,
                                const float* out, const float* grad_out, const int* img_idx, const float* weight_delta, int fixed_img,
                                float* grad_x, float* grad_weight_delta, float* grad_bias, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_calib_sigmoid_backward<<<div_up((long long)nr_rays * 32, kThreads), kThreads, 0, ST>>>(
        nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n, x, out, grad_out, img_idx, weight_delta, fixed_img, grad_x,
        grad_weight_delta, grad_bias);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
}  // extern "C"

// ---------------------------------------------------------------------------------------------- curvature loss
// SDF.get_sdf_and_curvature_1d_precomputed_gradient_normal_based (permuto_sdf_py/models/models.py:261-294):
//   tangent = cross(normalize(g), normalize(rand));  points_shifted = points + eps * tangent          (k_curv_shift)
//   curvature = acos(clamp(normalize(g) . normalize(g_shifted), -1 + 1e-6, 1 - 1e-6)) / pi               (k_curv_forward)
// and the mean of the curvature over the valid samples as the loss term (train_permuto_sdf.py:362-366). The element-wise
// chain (3 normalisations, cross, dot, clamp, acos, mean) is ~18 launches forward and ~30 backward in PyTorch.
namespace {
__device__ __forceinline__ void normalize3(float x, float y, float z, float& nx, float& ny, float& nz, float& inv, bool& ok) {
    // same operations as F.normalize (no FMA contraction, true divisions): the curvature term is ill-conditioned in these roundings
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    ok = n > 1e-12f;                               // F.normalize(eps = 1e-12): x / max(|x|, eps)
    const float den = fmaxf(n, 1e-12f);
    inv = 1.0f / den;
    nx = __fdiv_rn(x, den); ny = __fdiv_rn(y, den); nz = __fdiv_rn(z, den);
}
__global__ void __launch_bounds__(kThreads)
k_curv_shift(int n, const float* __restrict__ points, const float* __restrict__ g, const float* __restrict__ rnd, float eps,
             float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float nx, ny, nz, rx, ry, rz, inv;
    bool ok;
    normalize3(g[3 * i], g[3 * i + 1], g[3 * i + 2], nx, ny, nz, inv, ok);
    normalize3(rnd[3 * i], rnd[3 * i + 1], rnd[3 * i + 2], rx, ry, rz, inv, ok);
    out[3 * i] = points[3 * i] + (ny * rz - nz * ry) * eps;
    out[3 * i + 1] = points[3 * i + 1] + (nz * rx - nx * rz) * eps;
    out[3 * i + 2] = points[3 * i + 2] + (nx * ry - ny * rx) * eps;
}
// curv [n] (0 for rows >= *nr_valid_dev) and loss_sum += sum of the valid rows
__global__ void __launch_bounds__(kThreads)
k_curv_forward(int n, const float* __restrict__ g, const float* __restrict__ gs, const int* __restrict__ nr_valid_dev,
               float* __restrict__ curv, float* __restrict__ loss_sum) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int nv = nr_valid_dev ? min(nr_valid_dev[0], n) : n;
    float c = 0.0f;
    if (i < nv) {
        float ax, ay, az, bx, by, bz, inv;
        bool ok;
        normalize3(g[3 * i], g[3 * i + 1], g[3 * i + 2], ax, ay, az, inv, ok);
        normalize3(gs[3 * i], gs[3 * i + 1], gs[3 * i + 2], bx, by, bz, inv, ok);
        const float dot = __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
        const float d = fminf(fmaxf(dot, -1.0f + 1e-6f), 1.0f - 1e-6f);
        c = acosf(d) * 0.3183098861837907f;
    }
    if (i < n) curv[i] = c;
    const float s = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && s != 0.0f) atomicAdd(loss_sum, s);
}
// d (scale * sum_valid curv) / d g, d gs ; scale = *g_loss_dev * (by_count ? 1 / max(nr_valid, 1) : 1)
__global__ void __launch_bounds__(kThreads)
k_curv_backward(int n, const float* __restrict__ g, const float* __restrict__ gs, const int* __restrict__ nr_valid_dev,
                const float* __restrict__ g_loss_dev, float scale, float* __restrict__ gg, float* __restrict__ ggs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int nv = nr_valid_dev ? min(nr_valid_dev[0], n) : n;
    float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (i < nv) {
        float ax, ay, az, bx, by, bz, ia, ib;
        bool oka, okb;
        normalize3(g[3 * i], g[3 * i + 1], g[3 * i + 2], ax, ay, az, ia, oka);
        normalize3(gs[3 * i], gs[3 * i + 1], gs[3 * i + 2], bx, by, bz, ib, okb);
        const float d = __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
        if (d >= -1.0f + 1e-6f && d <= 1.0f - 1e-6f) {          // clamp passes the gradient inside the range (bounds included)
            const float up = (g_loss_dev ? g_loss_dev[0] : 1.0f) * scale / (float)(nr_valid_dev ? max(nv, 1) : 1);
            const float k = -up * 0.3183098861837907f / sqrtf(1.0f - d * d);     // d acos(d) / pi
            // d d / d g = (b - a (a.b)) / |g| when |g| > eps, else b / eps
            o[0] = k * (oka ? (bx - ax * d) : bx) * ia; o[1] = k * (oka ? (by - ay * d) : by) * ia; o[2] = k * (oka ? (bz - az * d) : bz) * ia;
            o[3] = k * (okb ? (ax - bx * d) : ax) * ib; o[4] = k * (okb ? (ay - by * d) : ay) * ib; o[5] = k * (okb ? (az - bz * d) : az) * ib;
        }
    }
    gg[3 * i] = o[0]; gg[3 * i + 1] = o[1]; gg[3 * i + 2] = o[2];
    ggs[3 * i] = o[3]; ggs[3 * i + 1] = o[4]; ggs[3 * i + 2] = o[5];
}
}  // namespace

extern "C" {
int psdf_curvature_shift_points(int n, const float* points, const float* sdf_grad, const float* rand_dirs, float eps, float* out,
                                void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_curv_shift<<<div_up(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n, points, sdf_grad, rand_dirs, eps, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_curvature_loss_forward(int n, const float* sdf_grad, const float* sdf_grad_shifted, const int* nr_valid_dev, float* curvature,
                                float* loss_sum, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_curv_forward<<<div_up(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n, sdf_grad, sdf_grad_shifted, nr_valid_dev, curvature, loss_sum);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_curvature_loss_backward(int n, const float* sdf_grad, const float* sdf_grad_shifted, const int* nr_valid_dev,
                                 const float* g_loss_dev, float scale, float* grad_sdf_grad, float* grad_sdf_grad_shifted, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_curv_backward<<<div_up(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n, sdf_grad, sdf_grad_shifted, nr_valid_dev, g_loss_dev, scale,
                                                                               grad_sdf_grad, grad_sdf_grad_shifted);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
}  // extern "C"
