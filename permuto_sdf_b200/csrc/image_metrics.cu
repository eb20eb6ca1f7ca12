// Image metrics of the reference's evaluate_psnr.py, sm_90a: per-image PSNR and SSIM as piq.psnr / piq.ssim compute them at
// data_range = 1 (kernel 11, sigma 1.5, k1 0.01, k2 0.03, piq's average-pool downsampling), on fp32 images in device memory.
//
// Inputs are read as fp32; everything after the optional quantization (an fp32 round trip through 8 bits, as the PNGs the reference scores)
// is fp64: the mask product, the pooling, the window sums, the moments, the formulas and the means. Each CTA writes one fp64 partial sum and
// a second kernel adds an image's partials in a fixed order, with no float atomics, so a call gives the same bits on every run. The number
// of partials depends only on the image size, not on the device.
//
//   k_im_psnr        sum over (pixel, channel) of (x - y)^2, one partial per CTA                     grid (psnr_parts(H W), B), 256 threads
//   k_im_ssim        one CTA per 32 x 8 tile of SSIM positions of one image, every channel:          grid (tiles, B), 256 threads
//                    stage the pooled, quantized and masked x and y of the tile and its 10-pixel halo in shared memory, the horizontal
//                    11-tap pass into the five moment rows (x, y, xx, yy, xy), the vertical pass and ss; one partial per CTA
//   k_im_finish      out[b] = the fixed-order sum of image b's partials, turned into dB (PSNR) or a mean (SSIM)   one CTA per image
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kWin = 11, kHalf = 5;                       // piq's kernel_size and (kernel_size - 1) / 2
constexpr double kSigma = 1.5, kC1 = 0.01 * 0.01, kC2 = 0.03 * 0.03, kEps = 1e-8;
constexpr int kTileW = 32, kTileH = kThreads / kTileW;    // SSIM positions per CTA: one per thread
constexpr int kStageW = kTileW + kWin - 1, kStageH = kTileH + kWin - 1;
constexpr int kPsnrPixelsPerThread = 8, kPsnrMaxParts = 1024;
constexpr long long kIntMax = 0x7fffffffLL;
#define ST ((cudaStream_t)stream)

struct Img {
    int B, C, H, W;
    const float* x;
    const float* y;
    const float* mask;     // [B, H, W] or nullptr
    int x_nhwc, y_nhwc, quantize_x;
};

// piq's downsampling factor f = max(1, round(min(H, W) / 256)), with Python's round (half to even): min(H, W) / 256 is exact in fp64
inline int pool_factor(long long H, long long W) {
    const long long m = H < W ? H : W;
    long long q = m / 256, r = m % 256;
    if (r > 128 || (r == 128 && (q & 1))) q++;
    return q > 1 ? (int)q : 1;
}

inline int psnr_parts(long long HW) {
    const long long n = (HW + (long long)kThreads * kPsnrPixelsPerThread - 1) / ((long long)kThreads * kPsnrPixelsPerThread);
    return (int)(n < kPsnrMaxParts ? (n > 0 ? n : 1) : kPsnrMaxParts);
}

inline long long ssim_tiles(long long Hp, long long Wp) {
    if (Hp < kWin || Wp < kWin) return 0;
    return ((Wp - kWin + kTileW) / kTileW) * ((Hp - kWin + kTileH) / kTileH);
}

__device__ __forceinline__ long long offset(bool nhwc, const Img& I, int b, int c, long long yy, long long xx) {
    return nhwc ? (((long long)b * I.H + yy) * I.W + xx) * I.C + c : (((long long)b * I.C + c) * I.H + yy) * I.W + xx;
}

// create_my_images' PNG round trip, in fp32: min(255, max(0, rne(x * 255))) / 255
__device__ __forceinline__ float quantize(float v) {
    return __fdiv_rn(fminf(255.0f, fmaxf(0.0f, rintf(__fmul_rn(v, 255.0f)))), 255.0f);
}

// the two values at (b, c, yy, xx) after the quantization of x and the mask: x m and y m in fp64 (exact products of fp32 values)
__device__ __forceinline__ void load_pair(const Img& I, int b, int c, long long yy, long long xx, double m, double& xv, double& yv) {
    float a = __ldg(I.x + offset(I.x_nhwc, I, b, c, yy, xx));
    if (I.quantize_x) a = quantize(a);
    xv = (double)a * m;
    yv = (double)__ldg(I.y + offset(I.y_nhwc, I, b, c, yy, xx)) * m;
}

__device__ __forceinline__ double mask_at(const Img& I, int b, long long yy, long long xx) {
    return I.mask ? (double)__ldg(I.mask + ((long long)b * I.H + yy) * I.W + xx) : 1.0;
}

// sum of v over the CTA, in a fixed order: a butterfly within each warp, then warp 0 adds the warps' sums in warp order
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double warp_sum[kWarps];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kWarps; w++) s += warp_sum[w];
    return s;                                  // valid in thread 0
}

__global__ void __launch_bounds__(kThreads) k_im_psnr(Img I, double* __restrict__ parts) {
    const int b = blockIdx.y;
    const long long HW = (long long)I.H * I.W;
    double acc = 0.0;
    for (long long p = (long long)blockIdx.x * kThreads + threadIdx.x; p < HW; p += (long long)gridDim.x * kThreads) {
        const long long yy = p / I.W, xx = p - yy * I.W;
        const double m = mask_at(I, b, yy, xx);
        for (int c = 0; c < I.C; c++) {
            double xv, yv;
            load_pair(I, b, c, yy, xx, m, xv, yv);
            const double d = xv - yv;
            acc += d * d;
        }
    }
    const double s = block_sum(acc);
    if (threadIdx.x == 0) parts[(long long)b * gridDim.x + blockIdx.x] = s;
}

// one CTA per tile of kTileH x kTileW SSIM positions (valid-mode window origins) of image blockIdx.y, all channels
__global__ void __launch_bounds__(kThreads) k_im_ssim(Img I, int f, int Hp, int Wp, int tiles_x, double* __restrict__ parts) {
    __shared__ double g[kWin];
    __shared__ double sx[kStageH][kStageW], sy[kStageH][kStageW];
    __shared__ double h[5][kStageH][kTileW];
    const int b = blockIdx.y;
    const int ty0 = (blockIdx.x / tiles_x) * kTileH, tx0 = (blockIdx.x % tiles_x) * kTileW;
    const int tid = threadIdx.x;
    if (tid < kWin) {
        // piq's gaussian_filter is the outer product of this 1-D window with itself, normalised to sum 1; so is the product of two
        // normalised 1-D windows
        double s = 0.0, gi = 0.0;
        for (int i = 0; i < kWin; i++) {
            const double c = (double)(i - kHalf);
            const double e = exp(-(c * c) / (2.0 * kSigma * kSigma));
            s += e;
            if (i == tid) gi = e;
        }
        g[tid] = gi / s;
    }
    const double inv_area = 1.0 / ((double)f * f);
    const int oy = tid / kTileW, ox = tid % kTileW;
    const bool valid = ty0 + oy <= Hp - kWin && tx0 + ox <= Wp - kWin;
    double acc = 0.0;
    for (int c = 0; c < I.C; c++) {
        // stage: average of the f x f block of masked values under each pooled pixel (F.avg_pool2d(., f)); outside the image: 0
        for (int k = tid; k < kStageH * kStageW; k += kThreads) {
            const int r = k / kStageW, q = k % kStageW;
            const int py = ty0 + r, px = tx0 + q;
            double ax = 0.0, ay = 0.0;
            if (py < Hp && px < Wp) {
                for (int dy = 0; dy < f; dy++) {
                    const long long yy = (long long)py * f + dy;
                    for (int dx = 0; dx < f; dx++) {
                        const long long xx = (long long)px * f + dx;
                        double xv, yv;
                        load_pair(I, b, c, yy, xx, mask_at(I, b, yy, xx), xv, yv);
                        ax += xv;
                        ay += yv;
                    }
                }
                ax *= inv_area;
                ay *= inv_area;
            }
            sx[r][q] = ax;
            sy[r][q] = ay;
        }
        __syncthreads();
        // horizontal pass: the 11-tap sums of x, y, x^2, y^2 and x y along each staged row
        for (int k = tid; k < kStageH * kTileW; k += kThreads) {
            const int r = k / kTileW, q = k % kTileW;
            double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0, m4 = 0.0;
#pragma unroll
            for (int j = 0; j < kWin; j++) {
                const double a = sx[r][q + j], e = sy[r][q + j], w = g[j];
                m0 += w * a;
                m1 += w * e;
                m2 += w * (a * a);
                m3 += w * (e * e);
                m4 += w * (a * e);
            }
            h[0][r][q] = m0; h[1][r][q] = m1; h[2][r][q] = m2; h[3][r][q] = m3; h[4][r][q] = m4;
        }
        __syncthreads();
        // vertical pass and piq's formulas at this thread's position
        if (valid) {
            double mx = 0.0, my = 0.0, exx = 0.0, eyy = 0.0, exy = 0.0;
#pragma unroll
            for (int i = 0; i < kWin; i++) {
                const double w = g[i];
                mx += w * h[0][oy + i][ox];
                my += w * h[1][oy + i][ox];
                exx += w * h[2][oy + i][ox];
                eyy += w * h[3][oy + i][ox];
                exy += w * h[4][oy + i][ox];
            }
            // rounded as written, with no contraction: for x = y both fractions are then exactly 1
            const double mxx = __dmul_rn(mx, mx), myy = __dmul_rn(my, my), mxy = __dmul_rn(mx, my);
            const double sxx = __dsub_rn(exx, mxx), syy = __dsub_rn(eyy, myy), sxy = __dsub_rn(exy, mxy);
            const double cs = (2.0 * sxy + kC2) / __dadd_rn(__dadd_rn(sxx, syy), kC2);
            acc += (2.0 * mxy + kC1) / __dadd_rn(__dadd_rn(mxx, myy), kC1) * cs;
        }
        __syncthreads();                      // the next channel overwrites sx, sy and h
    }
    const double s = block_sum(acc);
    if (tid == 0) parts[(long long)b * gridDim.x + blockIdx.x] = s;
}

// out[b] from image b's n partials: psnr != 0: -10 log10(sum / count + 1e-8), else sum / count
__global__ void __launch_bounds__(kThreads) k_im_finish(int n, const double* __restrict__ parts, double count, int psnr, double* __restrict__ out) {
    const int b = blockIdx.x;
    double acc = 0.0;
    for (int k = threadIdx.x; k < n; k += kThreads) acc += parts[(long long)b * n + k];
    const double s = block_sum(acc);
    if (threadIdx.x == 0) out[b] = psnr ? -10.0 * log10(s / count + kEps) : s / count;
}

bool args_ok(int B, int C, int H, int W, const float* x, int x_nhwc, const float* y, int y_nhwc, int quantize_x, const double* out,
             const uint8_t* workspace) {
    return B >= 1 && B <= 65535 && C >= 1 && H >= 1 && W >= 1 && x && y && out && workspace && (x_nhwc == 0 || x_nhwc == 1) &&
           (y_nhwc == 0 || y_nhwc == 1) && (quantize_x == 0 || quantize_x == 1);
}
}  // namespace

extern "C" {

long long psdf_image_metrics_workspace_bytes(long long B, long long C, long long H, long long W) {
    if (B < 1 || C < 1 || H < 1 || W < 1) return PSDF_ERR_ARG;
    if (B > 65535 || C > kIntMax || H > kIntMax || W > kIntMax) return PSDF_ERR_UNSUPPORTED;
    const int f = pool_factor(H, W);
    const long long p = psnr_parts(H * W), t = ssim_tiles(H / f, W / f);
    return 8LL * B * (p > t ? p : t);
}

int psdf_image_psnr(int B, int C, int H, int W, const float* x, int x_nhwc, const float* y, int y_nhwc, const float* mask, int quantize_x,
                    double* out, uint8_t* workspace, void* stream) {
    if (!args_ok(B, C, H, W, x, x_nhwc, y, y_nhwc, quantize_x, out, workspace)) return PSDF_ERR_ARG;
    const Img I{B, C, H, W, x, y, mask, x_nhwc, y_nhwc, quantize_x};
    double* parts = reinterpret_cast<double*>(workspace);
    const int n = psnr_parts((long long)H * W);
    k_im_psnr<<<dim3(n, B), kThreads, 0, ST>>>(I, parts);
    k_im_finish<<<B, kThreads, 0, ST>>>(n, parts, (double)C * H * W, 1, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_image_ssim(int B, int C, int H, int W, const float* x, int x_nhwc, const float* y, int y_nhwc, const float* mask, int quantize_x,
                    double* out, uint8_t* workspace, void* stream) {
    if (!args_ok(B, C, H, W, x, x_nhwc, y, y_nhwc, quantize_x, out, workspace)) return PSDF_ERR_ARG;
    const int f = pool_factor(H, W), Hp = H / f, Wp = W / f;
    if (Hp < kWin || Wp < kWin) return PSDF_ERR_ARG;
    const Img I{B, C, H, W, x, y, mask, x_nhwc, y_nhwc, quantize_x};
    double* parts = reinterpret_cast<double*>(workspace);
    const int tiles_x = (Wp - kWin + kTileW) / kTileW;
    const int n = (int)ssim_tiles(Hp, Wp);
    k_im_ssim<<<dim3(n, B), kThreads, 0, ST>>>(I, f, Hp, Wp, tiles_x, parts);
    k_im_finish<<<B, kThreads, 0, ST>>>(n, parts, (double)C * (Hp - kWin + 1) * (Wp - kWin + 1), 0, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
