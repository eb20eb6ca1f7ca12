// Fused NeuS compositing + per-ray losses for training (sm_90a), forward and backward, one warp per ray.
//
// Replaces, in one kernel each way, what the reference runs as ~60 PyTorch element-wise launches plus 8 of its own
// kernels per iteration (volume_rendering_modules.py:129-176 `VolumeRenderingNeus.compute_weights` + `integrate`,
// volume_rendering_funcs.py:55-223, and the losses of train_permuto_sdf.py:349-353,380-383 /
// permuto_sdf_utils.py:43-51):
//   true_cos = dir . g ; iter_cos = -(relu(.5 - .5 c)(1-r) + relu(-c) r)
//   est_prev/next = sdf -/+ iter_cos dt / 2 ; alpha = clip((sig(prev s) - sig(next s) + 1e-5)/(sig(prev s) + 1e-5), 0, 1)
//   T_i = prod_{j<i} (1 - alpha_j + 1e-7) ; w = alpha T ; pred_rgb = sum w rgb ; w_sum = sum w ; bg_T = T_last
//   losses per ray: sum_c |gt_c - pred_c| * hit ; BCE(clip(w_sum, 1e-3, 1-1e-3), mask) ; sum_i (|g_i| - 1)^2
// The backward kernel re-derives alpha / T (saved) and returns d loss / d {sdf, g, rgb, inv_s} for
//   loss = mean_{R,3}(rgb term) + w_eik mean_N(eik term) + w_mask mean_R(bce term).
// The transmittance recurrence runs as the same uniform serial chain as volrender.cu (left-to-right order).
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

// Optional extras of the direct (autograd-free) training iteration (train.py Trainer._iteration_direct), all off by default:
//  * colour head: `rgb` holds the RAW output x of the colour network; colour = sigmoid(x (1 + weight_delta[img]) + bias[img])
//    (Colorcal.calib_RGB_samples_packed + sigmoid, models.py:395-414,677-741), identity calibration for img == fixed_img / img_idx == NULL;
//    the backward then returns d loss / d x in g_rgb and accumulates the per-image parameter gradients;
//  * curvature term: with gs = d sdf/dx at the shifted points the backward adds d (curv_scale * sum_i curvature_i) / d g to g_grad and
//    writes d / d gs to ggs (rgb_misc.cu k_curv_backward folded in);
//  * tail: rows [nr_samples_dev[0], n_rows) of the gradient buffers are zero-filled by extra blocks (static-capacity containers),
//    so that the caller needs no memset.
struct NeusExt {
    unsigned long long* fx;         // deterministic mode: DetBufs::neus (calibration and inv_s gradients in fixed point), else NULL
    int head;                       // 1: rgb is the raw network output
    const int* img_idx;             // [R] or NULL
    const float* weight_delta;      // [nr_imgs,3]
    const float* bias;              // [nr_imgs,3]
    int fixed_img;
    float* g_weight_delta;          // (+=) or NULL
    float* g_bias;                  // (+=)
    const float* gs;                // [N,3] shifted-point gradients or NULL (no curvature term)
    float* ggs;                     // [N,3] (=)
    float curv_scale;               // weight of the curvature MEAN (divided by the sample count on the device)
    const float* curv_scale_dev;    // optional device multiplier [1]
    int n_rows;                     // rows of the gradient buffers (tail zero-fill), 0: no tail handling
    const int* nr_valid_dev;        // [1] rows covered by rays (the container's own sample count); NULL: all n_rows are covered
    int ray_blocks;                 // blocks [0, ray_blocks) walk rays, the rest zero the tail
};
__device__ __forceinline__ float sigmoid_exact(float v) { return 1.0f / (1.0f + expf(-v)); }
__device__ __forceinline__ void normalize3n(float x, float y, float z, float& nx, float& ny, float& nz, float& inv, bool& ok) {
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    ok = n > 1e-12f;
    const float den = fmaxf(n, 1e-12f);
    inv = 1.0f / den;
    nx = __fdiv_rn(x, den); ny = __fdiv_rn(y, den); nz = __fdiv_rn(z, den);
}

struct NeusSample {
    float alpha, q, pc, nc, prev, next, ic_d;   // ic_d = d iter_cos / d true_cos
};
__device__ __forceinline__ NeusSample neus_alpha(float sdf, float gx, float gy, float gz, float dx, float dy, float dz, float dt, float s,
                                                 float r) {
    NeusSample o;
    float tc = dx * gx + dy * gy + dz * gz;
    float a = fmaxf(-tc * 0.5f + 0.5f, 0.0f), b = fmaxf(-tc, 0.0f);
    float ic = -(a * (1.0f - r) + b * r);
    o.ic_d = (tc < 1.0f ? 0.5f * (1.0f - r) : 0.0f) + (tc < 0.0f ? r : 0.0f);
    o.next = sdf + ic * dt * 0.5f;
    o.prev = sdf - ic * dt * 0.5f;
    o.pc = sigmoidf_(o.prev * s);
    o.nc = sigmoidf_(o.next * s);
    o.q = (o.pc - o.nc + 1e-5f) / (o.pc + 1e-5f);
    o.alpha = fminf(fmaxf(o.q, 0.0f), 1.0f);
    return o;
}

// kRender: the forward of a rendered frame (psdf_neus_render_forward). The alpha / transmittance chain and the colour head are the
// training kernel's code; there are no loss terms and nothing is stored per sample (gt_rgb, gt_mask, hit, alpha_out, T_out, w_out, bg_T
// and ray_loss are not read), and the warp also accumulates sum w grad in the order of sum w rgb. Per ray it writes pred_rgb, w_sum,
// pred_normals = F.normalize(sum w grad) (eps 1e-12) and, with bg_rgb, pred_rgb_bg = T_last bg_rgb.
template <bool kRender>
__global__ void __launch_bounds__(kThreads)
k_neus_forward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n, const float* __restrict__ sdf,
               const float* __restrict__ grad, const float* __restrict__ rgb, const float* __restrict__ dirs, const float* __restrict__ dt_,
               const float* __restrict__ inv_s_dev, float cos_anneal, const float* __restrict__ cos_anneal_dev, const float* __restrict__ gt_rgb, const float* __restrict__ gt_mask,
               const uint8_t* __restrict__ hit, const float* __restrict__ bg_rgb, float* __restrict__ alpha_out, float* __restrict__ T_out, float* __restrict__ w_out,
               float* __restrict__ pred_rgb, float* __restrict__ w_sum, float* __restrict__ bg_T, float* __restrict__ ray_loss /* [R,3] */,
               NeusExt ext, float* __restrict__ pred_rgb_bg, float* __restrict__ pred_normals) {
    int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    RayRange rr = ray_range(ray, start_end, equal, fixed_n);
    bool skip = (rr.end > max_nr_samples) || (rr.n == 0);
    const float s = fminf(fmaxf(inv_s_dev[0], 1e-6f), 1e6f);
    if (cos_anneal_dev) cos_anneal = cos_anneal_dev[0];
    float hw[3] = {1.f, 1.f, 1.f}, hb[3] = {0.f, 0.f, 0.f};
    if (ext.head && ext.img_idx) {
        const int im = ext.img_idx[ray];
        if (im != ext.fixed_img) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) { hw[ch] = 1.0f + ext.weight_delta[3 * im + ch]; hb[ch] = ext.bias ? ext.bias[3 * im + ch] : 0.0f; }
        }
    }
    float T = 1.0f, ax = 0.f, ay = 0.f, az = 0.f, ws = 0.f, eik = 0.f;
    float nx = 0.f, ny = 0.f, nz = 0.f;     // render mode: sum w grad
    if (!skip) {
        for (int base = 0; base < rr.n; base += 32) {
            int i = base + lane;
            float al = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
            float gx = 0.f, gy = 0.f, gz = 0.f;
            if (i < rr.n) {
                int k = rr.start + i;
                gx = grad[3 * k]; gy = grad[3 * k + 1]; gz = grad[3 * k + 2];
                NeusSample ns = neus_alpha(sdf[k], gx, gy, gz, dirs[3 * k], dirs[3 * k + 1], dirs[3 * k + 2], dt_[k], s, cos_anneal);
                al = ns.alpha;
                cr = rgb[3 * k]; cg = rgb[3 * k + 1]; cb = rgb[3 * k + 2];
                if (ext.head) { cr = sigmoid_exact(cr * hw[0] + hb[0]); cg = sigmoid_exact(cg * hw[1] + hb[1]); cb = sigmoid_exact(cb * hw[2] + hb[2]); }
                if constexpr (!kRender) {
                    float nrm = sqrtf(gx * gx + gy * gy + gz * gz) - 1.0f;
                    eik += nrm * nrm;
                    alpha_out[k] = al;
                }
            }
            float myT = 1.0f;
            int cnt = min(32, rr.n - base);
            for (int k = 0; k < cnt; k++) {
                float ak = __shfl_sync(kFull, al, k);
                if (lane == k) myT = T;
                float wk = ak * T;
                ax = fmaf(wk, __shfl_sync(kFull, cr, k), ax);
                ay = fmaf(wk, __shfl_sync(kFull, cg, k), ay);
                az = fmaf(wk, __shfl_sync(kFull, cb, k), az);
                if constexpr (kRender) {
                    nx = fmaf(wk, __shfl_sync(kFull, gx, k), nx);
                    ny = fmaf(wk, __shfl_sync(kFull, gy, k), ny);
                    nz = fmaf(wk, __shfl_sync(kFull, gz, k), nz);
                }
                ws += wk;
                if (base + k < rr.n - 1) T *= (1.0f - ak + 1e-7f);
            }
            if constexpr (!kRender) {
                if (i < rr.n) { T_out[rr.start + i] = myT; if (w_out) w_out[rr.start + i] = al * myT; }
            }
        }
        if constexpr (!kRender) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) eik += __shfl_xor_sync(kFull, eik, o);
        }
    }
    if (lane == 0) {
        if (bg_rgb) { ax = fmaf(T, bg_rgb[3 * ray], ax); ay = fmaf(T, bg_rgb[3 * ray + 1], ay); az = fmaf(T, bg_rgb[3 * ray + 2], az); }
        pred_rgb[3 * ray] = ax; pred_rgb[3 * ray + 1] = ay; pred_rgb[3 * ray + 2] = az;
        w_sum[ray] = ws;
        if constexpr (kRender) {
            if (bg_rgb && pred_rgb_bg) {
#pragma unroll
                for (int c = 0; c < 3; c++) pred_rgb_bg[3 * ray + c] = T * bg_rgb[3 * ray + c];
            }
            // F.normalize(v, dim=1): v / max(||v||_2, 1e-12)
            const float den = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-12f);
            pred_normals[3 * ray] = nx / den; pred_normals[3 * ray + 1] = ny / den; pred_normals[3 * ray + 2] = nz / den;
            return;
        }
        bg_T[ray] = T;
        float h = hit ? (hit[ray] ? 1.0f : 0.0f) : 1.0f;
        float l1 = (fabsf(gt_rgb[3 * ray] - ax) + fabsf(gt_rgb[3 * ray + 1] - ay) + fabsf(gt_rgb[3 * ray + 2] - az)) * h;
        float bce = 0.0f;
        if (gt_mask) {
            float p = fminf(fmaxf(ws, 1e-3f), 1.0f - 1e-3f), m = gt_mask[ray];
            bce = -(m * fmaxf(logf(p), -100.0f) + (1.0f - m) * fmaxf(logf(1.0f - p), -100.0f));
        }
        ray_loss[3 * ray] = l1; ray_loss[3 * ray + 1] = bce; ray_loss[3 * ray + 2] = eik;
    }
}

// scale_rgb = g_total / (3R), scale_mask = g_total w_mask / R, scale_eik = g_total w_eik / N
__global__ void __launch_bounds__(kThreads)
k_neus_backward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n, const float* __restrict__ sdf,
                const float* __restrict__ grad, const float* __restrict__ rgb, const float* __restrict__ dirs, const float* __restrict__ dt_,
                const float* __restrict__ inv_s_dev, float cos_anneal, const float* __restrict__ cos_anneal_dev, const float* __restrict__ gt_rgb, const float* __restrict__ gt_mask,
                const uint8_t* __restrict__ hit, const float* __restrict__ bg_rgb, const float* __restrict__ alpha_in,
                const float* __restrict__ T_in, const float* __restrict__ pred_rgb, const float* __restrict__ w_sum,
                const float* __restrict__ bg_T, const float* __restrict__ g_total_dev, float scale_rgb,
                float scale_mask, float scale_eik, const int* __restrict__ nr_samples_dev, float* __restrict__ g_sdf, float* __restrict__ g_grad, float* __restrict__ g_rgb,
                float* __restrict__ g_bg_rgb, float* __restrict__ g_inv_s, NeusExt ext) {
    if (ext.n_rows > 0 && (int)blockIdx.x >= ext.ray_blocks) {
        // tail blocks: rows past the device-side sample count belong to no ray and must carry zero gradients
        const int nv = ext.nr_valid_dev ? min(max(ext.nr_valid_dev[0], 0), ext.n_rows) : ext.n_rows;
        for (int i = nv + (blockIdx.x - ext.ray_blocks) * blockDim.x + threadIdx.x; i < ext.n_rows; i += (gridDim.x - ext.ray_blocks) * blockDim.x) {
            g_sdf[i] = 0.f;
#pragma unroll
            for (int c = 0; c < 3; c++) { g_grad[3 * i + c] = 0.f; g_rgb[3 * i + c] = 0.f; if (ext.ggs) ext.ggs[3 * i + c] = 0.f; }
        }
        return;
    }
    int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    RayRange rr = ray_range(ray, start_end, equal, fixed_n);
    const bool skip = (rr.end > max_nr_samples) || (rr.n == 0);
    if (skip && !bg_rgb) return;
    float hw[3] = {1.f, 1.f, 1.f}, hb[3] = {0.f, 0.f, 0.f};
    int him = -1;
    if (ext.head && ext.img_idx) {
        him = ext.img_idx[ray];
        if (him != ext.fixed_img) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) { hw[ch] = 1.0f + ext.weight_delta[3 * him + ch]; hb[ch] = ext.bias ? ext.bias[3 * him + ch] : 0.0f; }
        } else him = -1;
    }
    float hgw[3] = {0.f, 0.f, 0.f}, hgb[3] = {0.f, 0.f, 0.f};
    float curv_k = 0.0f;
    if (ext.gs) {
        const int cnt = nr_samples_dev ? max(nr_samples_dev[0], 1) : max(max_nr_samples, 1);
        curv_k = (g_total_dev ? g_total_dev[0] : 1.0f) * ext.curv_scale * (ext.curv_scale_dev ? ext.curv_scale_dev[0] : 1.0f) / (float)cnt;
    }
    const float gtot = g_total_dev ? g_total_dev[0] : 1.0f;
    const float s_raw = inv_s_dev[0];
    const float s = fminf(fmaxf(s_raw, 1e-6f), 1e6f);
    const bool s_active = (s_raw >= 1e-6f && s_raw <= 1e6f);
    if (cos_anneal_dev) cos_anneal = cos_anneal_dev[0];
    if (nr_samples_dev) scale_eik = scale_eik / (float)max(nr_samples_dev[0], 1);
    // upstream of the per-ray outputs
    float h = hit ? (hit[ray] ? 1.0f : 0.0f) : 1.0f;
    float gp[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float dlt = pred_rgb[3 * ray + c] - gt_rgb[3 * ray + c];
        gp[c] = gtot * scale_rgb * h * (dlt > 0.f ? 1.f : (dlt < 0.f ? -1.f : 0.f));
    }
    float gws = 0.0f;
    if (gt_mask) {
        float ws = w_sum[ray], m = gt_mask[ray];
        if (ws >= 1e-3f && ws <= 1.0f - 1e-3f) gws = gtot * scale_mask * (-(m / ws) + (1.0f - m) / (1.0f - ws));
    }
    const float ge = gtot * scale_eik;
    float gbg = 0.0f;   // d loss / d bg_T times bg_T
    if (bg_rgb) {
        float bt = bg_T[ray];
        gbg = (gp[0] * bg_rgb[3 * ray] + gp[1] * bg_rgb[3 * ray + 1] + gp[2] * bg_rgb[3 * ray + 2]) * bt;
        if (lane == 0 && g_bg_rgb) { g_bg_rgb[3 * ray] = gp[0] * bt; g_bg_rgb[3 * ray + 1] = gp[1] * bt; g_bg_rgb[3 * ray + 2] = gp[2] * bt; }
    }
    if (skip) return;
    // reverse sweep: S = sum_{k>i} gw_k w_k
    float S = 0.0f, gs_acc = 0.0f;
    const int nchunks = (rr.n + 31) / 32;
    for (int ch = nchunks - 1; ch >= 0; ch--) {
        int base = ch * 32;
        int i = base + lane;
        float al = 0.f, Ti = 0.f, gw = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
        int k = rr.start + i;
        float xr = 0.f, xg = 0.f, xb = 0.f;       // raw network outputs (colour head)
        if (i < rr.n) {
            al = alpha_in[k]; Ti = T_in[k];
            cr = rgb[3 * k]; cg = rgb[3 * k + 1]; cb = rgb[3 * k + 2];
            if (ext.head) {
                xr = cr; xg = cg; xb = cb;
                cr = sigmoid_exact(xr * hw[0] + hb[0]); cg = sigmoid_exact(xg * hw[1] + hb[1]); cb = sigmoid_exact(xb * hw[2] + hb[2]);
            }
            gw = gp[0] * cr + gp[1] * cg + gp[2] * cb + gws;
        }
        float gwww = gw * al * Ti;            // gw_i w_i
        float mySuffix = 0.0f;
        int cnt = min(32, rr.n - base);
        for (int j = cnt - 1; j >= 0; j--) {
            if (lane == j) mySuffix = S;
            S += __shfl_sync(kFull, gwww, j);
        }
        if (i < rr.n) {
            // d loss / d alpha_i : own weight + all later transmittances (the last sample does not enter any T)
            float b = fmaxf(1.0f - al + 1e-7f, 1e-6f);
            float ga = gw * Ti;
            if (i < rr.n - 1) ga -= (mySuffix + gbg) / b;
            float gx = grad[3 * k], gy = grad[3 * k + 1], gz = grad[3 * k + 2];
            float dx = dirs[3 * k], dy = dirs[3 * k + 1], dz = dirs[3 * k + 2];
            float dt = dt_[k];
            NeusSample ns = neus_alpha(sdf[k], gx, gy, gz, dx, dy, dz, dt, s, cos_anneal);
            float gq = (ns.q >= 0.0f && ns.q <= 1.0f) ? ga : 0.0f;
            float den = ns.pc + 1e-5f;
            float dq_dpc = (ns.nc) / (den * den);         // d/dpc [(pc - nc + e)/(pc + e)] = (nc)/(pc+e)^2
            float dq_dnc = -1.0f / den;
            float gpc = gq * dq_dpc * ns.pc * (1.0f - ns.pc);   // wrt (prev * s)
            float gnc = gq * dq_dnc * ns.nc * (1.0f - ns.nc);   // wrt (next * s)
            float gsdf = (gpc + gnc) * s;
            float gic = (gnc - gpc) * s * dt * 0.5f;
            float gtc = gic * ns.ic_d;
            gs_acc += gpc * ns.prev + gnc * ns.next;
            // eikonal term
            float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
            float ek = nrm > 0.f ? ge * 2.0f * (nrm - 1.0f) / nrm : 0.0f;
            g_sdf[k] = gsdf;
            float ogx = gtc * dx + ek * gx, ogy = gtc * dy + ek * gy, ogz = gtc * dz + ek * gz;
            if (ext.gs) {
                // curvature term: d (curv_k * acos(clamp(n . n_s)) / pi) / d {g, g_s}  (same expressions as rgb_misc.cu k_curv_backward)
                float ax_, ay_, az_, bx_, by_, bz_, ia, ib;
                bool oka, okb;
                const float sx = ext.gs[3 * k], sy = ext.gs[3 * k + 1], sz = ext.gs[3 * k + 2];
                normalize3n(gx, gy, gz, ax_, ay_, az_, ia, oka);
                normalize3n(sx, sy, sz, bx_, by_, bz_, ib, okb);
                const float d = __fadd_rn(__fadd_rn(__fmul_rn(ax_, bx_), __fmul_rn(ay_, by_)), __fmul_rn(az_, bz_));
                float o3 = 0.f, o4 = 0.f, o5 = 0.f;
                if (d >= -1.0f + 1e-6f && d <= 1.0f - 1e-6f) {
                    const float kk = -curv_k * 0.3183098861837907f / sqrtf(1.0f - d * d);
                    ogx += kk * (oka ? (bx_ - ax_ * d) : bx_) * ia; ogy += kk * (oka ? (by_ - ay_ * d) : by_) * ia; ogz += kk * (oka ? (bz_ - az_ * d) : bz_) * ia;
                    o3 = kk * (okb ? (ax_ - bx_ * d) : ax_) * ib; o4 = kk * (okb ? (ay_ - by_ * d) : ay_) * ib; o5 = kk * (okb ? (az_ - bz_ * d) : az_) * ib;
                }
                ext.ggs[3 * k] = o3; ext.ggs[3 * k + 1] = o4; ext.ggs[3 * k + 2] = o5;
            }
            g_grad[3 * k] = ogx; g_grad[3 * k + 1] = ogy; g_grad[3 * k + 2] = ogz;
            float wi = al * Ti;
            float q0 = gp[0] * wi, q1 = gp[1] * wi, q2 = gp[2] * wi;
            if (ext.head) {
                // through the sigmoid and the calibration: d / d x, per-image parameter gradients reduced over the ray
                const float v0 = q0 * cr * (1.0f - cr), v1 = q1 * cg * (1.0f - cg), v2 = q2 * cb * (1.0f - cb);
                hgw[0] += v0 * xr; hgw[1] += v1 * xg; hgw[2] += v2 * xb;
                hgb[0] += v0; hgb[1] += v1; hgb[2] += v2;
                q0 = v0 * hw[0]; q1 = v1 * hw[1]; q2 = v2 * hw[2];
            }
            g_rgb[3 * k] = q0; g_rgb[3 * k + 1] = q1; g_rgb[3 * k + 2] = q2;
        }
    }
    if (ext.head && him >= 0 && (ext.g_weight_delta || ext.g_bias)) {
        // each of the two gradients only where its buffer is given: a fixed-point total without a destination would never be flushed
        // (and cleared), and would reach the next launch's
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float sw = hgw[c], sb = hgb[c];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { sw += __shfl_xor_sync(kFull, sw, o); sb += __shfl_xor_sync(kFull, sb, o); }
            if (lane == 0 && ext.fx && him < kDetImages) {
                if (ext.g_weight_delta) fx_add(ext.fx + 3 * him + c, sw);
                if (ext.g_bias) fx_add(ext.fx + 3 * kDetImages + 3 * him + c, sb);
            } else if (lane == 0) {
                if (ext.g_weight_delta) atomicAdd(ext.g_weight_delta + 3 * him + c, sw);
                if (ext.g_bias) atomicAdd(ext.g_bias + 3 * him + c, sb);
            }
        }
    }
    if (g_inv_s) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) gs_acc += __shfl_xor_sync(kFull, gs_acc, o);
        if (lane == 0 && s_active && gs_acc != 0.0f) {
            if (ext.fx) fx_add(ext.fx + 6 * kDetImages, gs_acc);
            else atomicAdd(g_inv_s, gs_acc);
        }
    }
}
#define ST ((cudaStream_t)stream)
inline int ray_blocks(int nr_rays) { return div_up((long long)nr_rays * 32, kThreads); }
}  // namespace

extern "C" {
static int neus_forward_impl(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                             const float* grad, const float* rgb, const float* dirs, const float* dt, const float* inv_s_dev,
                             float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit,
                             const float* bg_rgb, float* alpha, float* transmittance, float* weights, float* pred_rgb, float* weights_sum,
                             float* bg_transmittance, float* ray_loss, const NeusExt& ext, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_neus_forward<false><<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n, sdf, grad, rgb, dirs,
                                                                   dt, inv_s_dev, cos_anneal_ratio, cos_anneal_dev, gt_rgb, gt_mask, hit, bg_rgb, alpha,
                                                                   transmittance, weights, pred_rgb, weights_sum, bg_transmittance, ray_loss, ext, nullptr,
                                                                   nullptr);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
static int neus_backward_impl(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                              const float* grad, const float* rgb, const float* dirs, const float* dt, const float* inv_s_dev,
                              float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit,
                              const float* bg_rgb, const float* alpha, const float* transmittance, const float* pred_rgb,
                              const float* weights_sum, const float* bg_transmittance, const float* g_total_dev, float scale_rgb,
                              float scale_mask, float scale_eik, const int* nr_samples_dev, float* g_sdf, float* g_grad, float* g_rgb,
                              float* g_bg_rgb, float* g_inv_s, NeusExt ext, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    const int rb = ray_blocks(nr_rays);
    ext.ray_blocks = rb;
    const DetBufs* dbuf = det_buffers();
    ext.fx = dbuf ? dbuf->neus : nullptr;
    const int tail_blocks = ext.n_rows > 0 ? min(div_up(ext.n_rows, kThreads), 132) : 0;
    k_neus_backward<<<rb + tail_blocks, kThreads, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n, sdf, grad, rgb, dirs, dt,
                                                          inv_s_dev, cos_anneal_ratio, cos_anneal_dev, gt_rgb, gt_mask, hit, bg_rgb, alpha,
                                                          transmittance, pred_rgb, weights_sum, bg_transmittance, g_total_dev, scale_rgb,
                                                          scale_mask, scale_eik, nr_samples_dev, g_sdf, g_grad, g_rgb, g_bg_rgb, g_inv_s, ext);
    PSDF_CHECK_LAUNCH();
    if (dbuf) {
        // deterministic mode: fixed-point totals -> the float gradients (+=); entries of images the buffers do not have stay zero and
        // are never written
        FxSegs F;
        if (ext.head) {
            F.add(dbuf->neus, ext.g_weight_delta, 3 * kDetImages);
            F.add(dbuf->neus + 3 * kDetImages, ext.g_bias, 3 * kDetImages);
        }
        F.add(dbuf->neus + 6 * kDetImages, g_inv_s, 1);
        if (fx_flush(F, ST) != 0) return PSDF_ERR_LAUNCH;
    }
    return PSDF_OK;
}
static NeusExt no_ext() {
    NeusExt e;
    e.fx = nullptr;
    e.head = 0; e.img_idx = nullptr; e.weight_delta = nullptr; e.bias = nullptr; e.fixed_img = -1; e.g_weight_delta = nullptr; e.g_bias = nullptr;
    e.gs = nullptr; e.ggs = nullptr; e.curv_scale = 0.f; e.curv_scale_dev = nullptr; e.n_rows = 0; e.ray_blocks = 0; e.nr_valid_dev = nullptr;
    return e;
}

int psdf_neus_render_loss_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                                  const float* grad, const float* rgb, const float* dirs, const float* dt, const float* inv_s_dev,
                                  float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit, const float* bg_rgb,
                                  float* alpha, float* transmittance, float* weights, float* pred_rgb, float* weights_sum, float* bg_transmittance,
                                  float* ray_loss, void* stream) {
    return neus_forward_impl(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, sdf, grad, rgb, dirs, dt, inv_s_dev, cos_anneal_ratio,
                             cos_anneal_dev, gt_rgb, gt_mask, hit, bg_rgb, alpha, transmittance, weights, pred_rgb, weights_sum, bg_transmittance,
                             ray_loss, no_ext(), stream);
}
int psdf_neus_render_loss_backward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                                   const float* grad, const float* rgb, const float* dirs, const float* dt, const float* inv_s_dev,
                                   float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit, const float* bg_rgb,
                                   const float* alpha, const float* transmittance, const float* pred_rgb, const float* weights_sum,
                                   const float* bg_transmittance, const float* g_total_dev,
                                   float scale_rgb, float scale_mask, float scale_eik, const int* nr_samples_dev, float* g_sdf, float* g_grad, float* g_rgb,
                                   float* g_bg_rgb, float* g_inv_s, void* stream) {
    return neus_backward_impl(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, sdf, grad, rgb, dirs, dt, inv_s_dev, cos_anneal_ratio,
                              cos_anneal_dev, gt_rgb, gt_mask, hit, bg_rgb, alpha, transmittance, pred_rgb, weights_sum, bg_transmittance,
                              g_total_dev, scale_rgb, scale_mask, scale_eik, nr_samples_dev, g_sdf, g_grad, g_rgb, g_bg_rgb, g_inv_s, no_ext(), stream);
}

// The same pair for the direct (autograd-free) iteration: the colour head (calibration + sigmoid) and the curvature term are folded in and
// the tail rows of the gradient buffers are zero-filled by the backward launch (see NeusExt). x_raw [N,3] is the colour network's linear
// output; img_idx / weight_delta may be NULL (no calibration), bias may be NULL (zero bias). weights may be NULL.
int psdf_neus_head_loss_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                                const float* grad, const float* x_raw, const float* dirs, const float* dt, const float* inv_s_dev,
                                float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit,
                                const int* img_idx, const float* weight_delta, const float* bias, int fixed_img, float* alpha,
                                float* transmittance, float* weights, float* pred_rgb, float* weights_sum, float* bg_transmittance,
                                float* ray_loss, void* stream) {
    NeusExt e = no_ext();
    e.head = 1; e.img_idx = weight_delta ? img_idx : nullptr; e.weight_delta = weight_delta; e.bias = bias; e.fixed_img = fixed_img;
    return neus_forward_impl(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, sdf, grad, x_raw, dirs, dt, inv_s_dev, cos_anneal_ratio,
                             cos_anneal_dev, gt_rgb, gt_mask, hit, nullptr, alpha, transmittance, weights, pred_rgb, weights_sum, bg_transmittance,
                             ray_loss, e, stream);
}
// -> g_sdf [n_rows], g_grad [n_rows,3] (compositing + eikonal + curvature terms), g_x [n_rows,3] (d loss / d raw colour output),
// g_grad_shifted [n_rows,3] (curvature term wrt the shifted-point gradients; grad_shifted may be NULL: no curvature term), per-image
// calibration gradients (+=, each may be NULL). curv_scale multiplies the curvature MEAN over nr_samples_dev[0] (or max_nr_samples) rows.
// nr_valid_dev [1] (static-capacity containers): rows [nr_valid_dev[0], n_rows) of the four gradient buffers are zero-filled.
int psdf_neus_head_loss_backward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                                 const float* grad, const float* x_raw, const float* dirs, const float* dt, const float* inv_s_dev,
                                 float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit,
                                 const int* img_idx, const float* weight_delta, const float* bias, int fixed_img, const float* alpha,
                                 const float* transmittance, const float* pred_rgb, const float* weights_sum, const float* bg_transmittance,
                                 float scale_rgb, float scale_mask, float scale_eik, const int* nr_samples_dev, const float* grad_shifted,
                                 float curv_scale, const float* curv_scale_dev, int n_rows, const int* nr_valid_dev, float* g_sdf, float* g_grad,
                                 float* g_x, float* g_grad_shifted, float* g_weight_delta, float* g_bias, void* stream) {
    NeusExt e = no_ext();
    e.head = 1; e.img_idx = weight_delta ? img_idx : nullptr; e.weight_delta = weight_delta; e.bias = bias; e.fixed_img = fixed_img;
    e.g_weight_delta = g_weight_delta; e.g_bias = g_bias;
    e.gs = grad_shifted; e.ggs = g_grad_shifted; e.curv_scale = curv_scale; e.curv_scale_dev = curv_scale_dev;
    if (grad_shifted && !g_grad_shifted) return PSDF_ERR_ARG;
    e.n_rows = nr_valid_dev ? n_rows : 0;        // without a device-side count the rays cover every row
    e.nr_valid_dev = nr_valid_dev;
    return neus_backward_impl(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, sdf, grad, x_raw, dirs, dt, inv_s_dev, cos_anneal_ratio,
                              cos_anneal_dev, gt_rgb, gt_mask, hit, nullptr, alpha, transmittance, pred_rgb, weights_sum, bg_transmittance,
                              nullptr, scale_rgb, scale_mask, scale_eik, nr_samples_dev, g_sdf, g_grad, g_x, nullptr, nullptr, e, stream);
}
// The head-loss pair of a scene without masks: bg_rgb [R,3] (the composited background colour) is blended in behind every ray, and the
// backward also returns g_bg_rgb [R,3] (=).
int psdf_neus_head_bg_loss_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                                   const float* grad, const float* x_raw, const float* dirs, const float* dt, const float* inv_s_dev,
                                   float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit,
                                   const int* img_idx, const float* weight_delta, const float* bias, int fixed_img, const float* bg_rgb,
                                   float* alpha, float* transmittance, float* weights, float* pred_rgb, float* weights_sum,
                                   float* bg_transmittance, float* ray_loss, void* stream) {
    NeusExt e = no_ext();
    e.head = 1; e.img_idx = weight_delta ? img_idx : nullptr; e.weight_delta = weight_delta; e.bias = bias; e.fixed_img = fixed_img;
    return neus_forward_impl(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, sdf, grad, x_raw, dirs, dt, inv_s_dev, cos_anneal_ratio,
                             cos_anneal_dev, gt_rgb, gt_mask, hit, bg_rgb, alpha, transmittance, weights, pred_rgb, weights_sum, bg_transmittance,
                             ray_loss, e, stream);
}
int psdf_neus_head_bg_loss_backward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf,
                                    const float* grad, const float* x_raw, const float* dirs, const float* dt, const float* inv_s_dev,
                                    float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb, const float* gt_mask, const uint8_t* hit,
                                    const int* img_idx, const float* weight_delta, const float* bias, int fixed_img, const float* bg_rgb,
                                    const float* alpha, const float* transmittance, const float* pred_rgb, const float* weights_sum,
                                    const float* bg_transmittance, float scale_rgb, float scale_mask, float scale_eik, const int* nr_samples_dev,
                                    const float* grad_shifted, float curv_scale, const float* curv_scale_dev, int n_rows, const int* nr_valid_dev,
                                    float* g_sdf, float* g_grad, float* g_x, float* g_grad_shifted, float* g_bg_rgb, float* g_weight_delta,
                                    float* g_bias, void* stream) {
    NeusExt e = no_ext();
    e.head = 1; e.img_idx = weight_delta ? img_idx : nullptr; e.weight_delta = weight_delta; e.bias = bias; e.fixed_img = fixed_img;
    e.g_weight_delta = g_weight_delta; e.g_bias = g_bias;
    e.gs = grad_shifted; e.ggs = g_grad_shifted; e.curv_scale = curv_scale; e.curv_scale_dev = curv_scale_dev;
    if (grad_shifted && !g_grad_shifted) return PSDF_ERR_ARG;
    e.n_rows = nr_valid_dev ? n_rows : 0;
    e.nr_valid_dev = nr_valid_dev;
    return neus_backward_impl(nr_rays, max_nr_samples, ray_start_end, equal, fixed_n, sdf, grad, x_raw, dirs, dt, inv_s_dev, cos_anneal_ratio,
                              cos_anneal_dev, gt_rgb, gt_mask, hit, bg_rgb, alpha, transmittance, pred_rgb, weights_sum, bg_transmittance,
                              nullptr, scale_rgb, scale_mask, scale_eik, nr_samples_dev, g_sdf, g_grad, g_x, g_bg_rgb, nullptr, e, stream);
}
// Forward-only compositing of a rendered frame (Trainer.render): the render mode of k_neus_forward, colour head on, no loss terms, nothing
// stored per sample. x_raw [N,3] is the colour network's linear output; img_idx / weight_delta may be NULL (no calibration), bias NULL is zero,
// bg_rgb [R,3] may be NULL (no background). pred_rgb_bg is written only with bg_rgb.
int psdf_neus_render_forward(int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n, const float* sdf, const float* grad,
                             const float* x_raw, const float* dirs, const float* dt, const float* inv_s_dev, float cos_anneal_ratio, const int* img_idx,
                             const float* weight_delta, const float* bias, int fixed_img, const float* bg_rgb, float* pred_rgb, float* pred_rgb_bg,
                             float* pred_normals, float* weights_sum, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    if (!pred_rgb || !pred_normals || !weights_sum || (bg_rgb && !pred_rgb_bg)) return PSDF_ERR_ARG;
    NeusExt e = no_ext();
    e.head = 1; e.img_idx = weight_delta ? img_idx : nullptr; e.weight_delta = weight_delta; e.bias = bias; e.fixed_img = fixed_img;
    k_neus_forward<true><<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n, sdf, grad, x_raw, dirs,
                                                                  dt, inv_s_dev, cos_anneal_ratio, nullptr, nullptr, nullptr, nullptr, bg_rgb, nullptr,
                                                                  nullptr, nullptr, pred_rgb, weights_sum, nullptr, nullptr, e, pred_rgb_bg, pred_normals);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
}  // extern "C"
