// SDF->density volume compositing, CDF / importance resampling and their hand-written backward
// kernels for sm_90a. One warp per ray over the packed sample container.
//
// Reference: kernels/permuto_sdf/VolumeRenderingGPU.cuh (one thread per ray, serial loop, strided
// accessor loads). Here every per-sample array is read/written with lane-contiguous (coalesced)
// accesses; recurrences whose floating-point order is observable (cumprod, cumsum, cdf, per-ray sums,
// weighted integration) run as a *uniform serial* recurrence: all 32 lanes replay the same scalar chain
// from warp-broadcast operands and lane k latches element k, so results are bit-identical to the
// reference's left-to-right order while memory traffic stays coalesced. Compiled with -fmad=false; FMAs
// are explicit where the reference build contracts (w*rgb accumulation, origin + z*dir).
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

#define RAY_PROLOGUE()                                                        \
    int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;                   \
    int lane = threadIdx.x & 31;                                              \
    if (ray >= nr_rays) return;                                               \
    RayRange rr = ray_range(ray, start_end, equal, fixed_n);                  \
    bool skip = (rr.end > max_nr_samples) || (rr.n == 0);

// VolumeRenderingGPU.cuh:371-422. alpha is already (1-alpha). T_i = prod_{j<i} a_j ; bg = T_{n-1}.
__global__ void __launch_bounds__(kThreads)
k_cumprod(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
          const float* __restrict__ alpha, float* __restrict__ T_out, float* __restrict__ bg_T) {
    RAY_PROLOGUE();
    if (skip) { if (lane == 0) bg_T[ray] = 1.0f; return; }
    float T = 1.0f;
    for (int base = 0; base < rr.n; base += 32) {
        int i = base + lane;
        float a = (i < rr.n) ? alpha[rr.start + i] : 1.0f;
        float mine = 1.0f;
        int cnt = min(32, rr.n - base);
        for (int k = 0; k < cnt; k++) {
            float ak = __shfl_sync(kFull, a, k);
            if (lane == k) mine = T;
            if (base + k < rr.n - 1) T = __fmul_rn(T, ak);
        }
        if (i < rr.n) T_out[rr.start + i] = mine;
    }
    if (lane == 0) bg_T[ray] = T;
}

// VolumeRenderingGPU.cuh:631-691 (forward or reverse inclusive cumsum) and :697-752 (exclusive cumsum = cdf)
template <bool EXCLUSIVE>
__global__ void __launch_bounds__(kThreads)
k_cumsum(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
         const float* __restrict__ vals, bool inverse, float* __restrict__ out) {
    RAY_PROLOGUE();
    if (skip) return;
    float acc = 0.0f;
    for (int base = 0; base < rr.n; base += 32) {
        int i = base + lane;
        int j = inverse ? (rr.end - 1 - i) : (rr.start + i);
        float v = (i < rr.n) ? vals[j] : 0.0f;
        float mine = 0.0f;
        int cnt = min(32, rr.n - base);
        for (int k = 0; k < cnt; k++) {
            float vk = __shfl_sync(kFull, v, k);
            if (EXCLUSIVE) { if (lane == k) mine = acc; acc = __fadd_rn(acc, vk); }
            else { acc = __fadd_rn(acc, vk); if (lane == k) mine = acc; }
        }
        if (i < rr.n) out[j] = mine;
    }
}

// VolumeRenderingGPU.cuh:566-628, val_dim == 1: serial sum, broadcast back to every sample of the ray
__global__ void __launch_bounds__(kThreads)
k_sum1(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
       const float* __restrict__ vals, float* __restrict__ sum_ray, float* __restrict__ sum_sample) {
    RAY_PROLOGUE();
    if (skip) { if (lane == 0) sum_ray[ray] = 0.0f; return; }
    float acc = 0.0f;
    for (int base = 0; base < rr.n; base += 32) {
        int i = base + lane;
        float v = (i < rr.n) ? vals[rr.start + i] : 0.0f;
        int cnt = min(32, rr.n - base);
        for (int k = 0; k < cnt; k++) acc = __fadd_rn(acc, __shfl_sync(kFull, v, k));
    }
    if (lane == 0) sum_ray[ray] = acc;
    for (int i = lane; i < rr.n; i += 32) sum_sample[rr.start + i] = acc;
}
// val_dim in {2,3,32}: lane v owns channel v and sums serially (same order as the reference)
__global__ void __launch_bounds__(kThreads)
k_sumD(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n, int D,
       const float* __restrict__ vals, float* __restrict__ sum_ray, float* __restrict__ sum_sample) {
    RAY_PROLOGUE();
    if (skip) { if (lane < D) sum_ray[ray * D + lane] = 0.0f; return; }
    float acc = 0.0f;
    if (lane < D) {
        const float* p = vals + (size_t)rr.start * D + lane;
#pragma unroll 4
        for (int i = 0; i < rr.n; i++) acc = __fadd_rn(acc, p[(size_t)i * D]);
        sum_ray[ray * D + lane] = acc;
        float* q = sum_sample + (size_t)rr.start * D + lane;
        for (int i = 0; i < rr.n; i++) q[(size_t)i * D] = acc;
    }
}

// VolumeRenderingGPU.cuh:425-481. acc_c = fma(w_i, v_ic, acc_c) left to right (FFMA in the reference build).
__global__ void __launch_bounds__(kThreads)
k_integrate(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
            const float* __restrict__ vals, const float* __restrict__ w, float* __restrict__ out) {
    RAY_PROLOGUE();
    if (skip) { if (lane < 3) out[3 * ray + lane] = 0.0f; return; }
    float ax = 0.0f, ay = 0.0f, az = 0.0f;
    for (int base = 0; base < rr.n; base += 32) {
        int i = base + lane;
        float wi = 0, x = 0, y = 0, z = 0;
        if (i < rr.n) {
            int s = rr.start + i;
            wi = w[s]; x = vals[3 * s]; y = vals[3 * s + 1]; z = vals[3 * s + 2];
        }
        int cnt = min(32, rr.n - base);
        for (int k = 0; k < cnt; k++) {
            float wk = __shfl_sync(kFull, wi, k);
            ax = __fmaf_rn(wk, __shfl_sync(kFull, x, k), ax);
            ay = __fmaf_rn(wk, __shfl_sync(kFull, y, k), ay);
            az = __fmaf_rn(wk, __shfl_sync(kFull, z, k), az);
        }
    }
    if (lane == 0) { out[3 * ray] = ax; out[3 * ray + 1] = ay; out[3 * ray + 2] = az; }
}

__device__ __forceinline__ float map_range(float v, float is, float ie, float os, float oe) {
    float c = fmaxf(is, fminf(ie, v));
    // os + ratio*(c-is): one FFMA in the reference build
    return __fmaf_rn(__fsub_rn(c, is), __fdiv_rn(__fsub_rn(oe, os), __fsub_rn(ie, is)), os);
}
__device__ __forceinline__ float sigmoid_ref(float x) { return (float)(1.0 / (1.0 + (double)expf(-x))); }

// VolumeRenderingGPU.cuh:490-564 ; alpha of the last sample of each ray stays 0
__global__ void __launch_bounds__(kThreads)
k_sdf2alpha(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, const float* __restrict__ ray_fixed_dt,
            const float* __restrict__ dt_, bool equal, int fixed_n, const float* __restrict__ sdf, float inv_s_in,
            bool dynamic_inv_s, float inv_s_mult, float* __restrict__ alpha) {
    RAY_PROLOGUE();
    if (skip) return;
    float inv_s = inv_s_in;
    if (dynamic_inv_s) inv_s = map_range(ray_fixed_dt[ray], 0.0001f, 0.01f, 1024.f, 64.f);
    inv_s = __fmul_rn(inv_s, inv_s_mult);
    for (int i = lane; i < rr.n; i += 32) {
        int s = rr.start + i;
        float a = 0.0f;
        if (i < rr.n - 1) {
            float dt = dt_[s];
            float prev = sdf[s], next = sdf[s + 1];
            float mid = __fmul_rn(__fadd_rn(prev, next), 0.5f);
            float cosv = __fdiv_rn(__fsub_rn(next, prev), fmaxf(1e-6f, dt));
            cosv = clampf(cosv, -1e3f, 0.0f);
            float h = __fmul_rn(cosv, dt);
            float pe = (float)((double)mid - (double)h * 0.5);
            float ne = (float)((double)mid + (double)h * 0.5);
            float pc = sigmoid_ref(__fmul_rn(pe, inv_s)), nc = sigmoid_ref(__fmul_rn(ne, inv_s));
            a = (float)(((double)__fsub_rn(pc, nc) + 1e-6) / ((double)pc + 1e-6));
        }
        alpha[s] = a;
    }
}

// first index in [imin,imax] whose cdf exceeds val (VolumeRenderingGPU.cuh:764-789, plus a guard for
// imax==imin where the reference loop never terminates)
__device__ __forceinline__ int cdf_search(const float* __restrict__ cdf, float val, int imin, int imax) {
    while (imax >= imin) {
        int imid = imin + (imax - imin) / 2;
        if (cdf[imid] > val) imax = imid; else imin = imid;
        if (imax - imin == 1) return imax;
        if (imax == imin) return imax;
    }
    return imax;
}
// VolumeRenderingGPU.cuh:793-946 ; lane i produces importance sample i (loops if nr_imp > 32). A ray with one sample has no
// cdf interval to draw from (the search would pair its sample with the previous ray's): it gets the samples of a skipped ray.
__global__ void __launch_bounds__(kThreads)
k_importance_sample(int nr_rays, const float* __restrict__ origins, const float* __restrict__ dirs, int max_nr_samples,
                    const int* __restrict__ start_end, const float* __restrict__ ray_fixed_dt, bool equal, int fixed_n,
                    const float* __restrict__ z, const float* __restrict__ cdf, int nr_imp, Pcg32 rng0, bool jitter,
                    float* __restrict__ o_pos, float* __restrict__ o_dirs, float* __restrict__ o_z) {
    rng0.resolve();
    RAY_PROLOGUE();
    int ist = ray * nr_imp;
    float ox = origins[3 * ray], oy = origins[3 * ray + 1], oz = origins[3 * ray + 2];
    float dx = dirs[3 * ray], dy = dirs[3 * ray + 1], dz = dirs[3 * ray + 2];
    float fixed_dt = ray_fixed_dt[ray];
    for (int i = lane; i < nr_imp; i += 32) {
        int s = ist + i;
        if (skip || rr.n == 1) {
            o_pos[3 * s] = 0; o_pos[3 * s + 1] = 0; o_pos[3 * s + 2] = 0;
            o_dirs[3 * s] = 0; o_dirs[3 * s + 1] = 0; o_dirs[3 * s + 2] = 0;
            o_z[s] = -1.0f;
            continue;
        }
        float du = (float)(1.0 / (double)(nr_imp + 1));
        float u = __fmaf_rn((float)i, du, du);
        if (jitter) {
            // the reference advances by `ray` before every draw, cumulatively (:872-878)
            Pcg32 rng = rng0;
            rng.advance((int64_t)(i + 1) * (int64_t)ray + (int64_t)i);
            float rnd = rng.next_float();
            float mov = (float)((double)du / 2.0);
            u = __fadd_rn(u, map_range(rnd, 0.0f, 1.0f, -mov, mov));
        }
        u = clampf(u, (float)(0.0 + 1e-6), (float)(1.0 - 1e-5));
        int imax = cdf_search(cdf, u, rr.start, rr.end - 1);
        int imin = max(imax - 1, 0);
        float cmax = cdf[imax], cmin = cdf[imin];
        float zmax = z[imax], zmin = z[imin];
        float zi = map_range(u, cmin, cmax, zmin, zmax);
        float dmin = __fsub_rn(zi, zmin), dmax = __fsub_rn(zmax, zi);
        if (dmin < dmax) { dmin = fminf(dmin, fixed_dt); zi = __fadd_rn(zmin, dmin); }
        else { dmax = fminf(dmax, fixed_dt); zi = __fsub_rn(zmax, dmax); }
        o_pos[3 * s] = __fmaf_rn(zi, dx, ox); o_pos[3 * s + 1] = __fmaf_rn(zi, dy, oy); o_pos[3 * s + 2] = __fmaf_rn(zi, dz, oz);
        o_dirs[3 * s] = dx; o_dirs[3 * s + 1] = dy; o_dirs[3 * s + 2] = dz;
        o_z[s] = zi;
    }
}

// One round of SDF-driven importance sampling (permuto_sdf_py/utils/sdf_utils.py importance_sampling_sdf_model: sdf2alpha ->
// clip -> cumprod(1 - alpha + 1e-7) -> weights -> per-ray normalisation -> cdf -> importance_sample) in ONE launch. Every
// intermediate keeps the arithmetic and the left-to-right order of the separate kernels / PyTorch ops it replaces (tests compare
// bit for bit); `cdf` is both scratch (un-normalised weights) and output.
__global__ void __launch_bounds__(kThreads)
k_importance_round(int nr_rays, const float* __restrict__ origins, const float* __restrict__ dirs, int max_nr_samples,
                   const int* __restrict__ start_end, const float* __restrict__ ray_fixed_dt, const float* __restrict__ dt_, bool equal,
                   int fixed_n, const float* __restrict__ z, const float* __restrict__ sdf, float inv_s_in, bool dynamic_inv_s,
                   float inv_s_mult, int nr_imp, Pcg32 rng0, bool jitter, float* __restrict__ cdf, float* __restrict__ o_pos,
                   float* __restrict__ o_dirs, float* __restrict__ o_z) {
    rng0.resolve();
    RAY_PROLOGUE();
    if (!skip) {
        float inv_s = inv_s_in;
        if (dynamic_inv_s) inv_s = map_range(ray_fixed_dt[ray], 0.0001f, 0.01f, 1024.f, 64.f);
        inv_s = __fmul_rn(inv_s, inv_s_mult);
        // alpha (k_sdf2alpha + clip) -> transmittance (k_cumprod of 1 - alpha + 1e-7) -> weight alpha * T
        float T = 1.0f;
        for (int base = 0; base < rr.n; base += 32) {
            const int i = base + lane, s = rr.start + i;
            float a = 0.0f;
            if (i < rr.n - 1) {
                const float dt = dt_[s];
                const float prev = sdf[s], next = sdf[s + 1];
                const float mid = __fmul_rn(__fadd_rn(prev, next), 0.5f);
                float cosv = __fdiv_rn(__fsub_rn(next, prev), fmaxf(1e-6f, dt));
                cosv = clampf(cosv, -1e3f, 0.0f);
                const float h = __fmul_rn(cosv, dt);
                const float pe = (float)((double)mid - (double)h * 0.5);
                const float ne = (float)((double)mid + (double)h * 0.5);
                const float pc = sigmoid_ref(__fmul_rn(pe, inv_s)), nc = sigmoid_ref(__fmul_rn(ne, inv_s));
                a = (float)(((double)__fsub_rn(pc, nc) + 1e-6) / ((double)pc + 1e-6));
            }
            a = fminf(fmaxf(a, 0.0f), 1.0f);
            const float b = (i < rr.n) ? __fadd_rn(__fsub_rn(1.0f, a), 1e-7f) : 1.0f;
            float mine = 1.0f;
            const int cnt = min(32, rr.n - base);
            for (int k = 0; k < cnt; k++) {
                const float bk = __shfl_sync(kFull, b, k);
                if (lane == k) mine = T;
                if (base + k < rr.n - 1) T = __fmul_rn(T, bk);
            }
            if (i < rr.n) cdf[s] = __fmul_rn(a, mine);
        }
        __syncwarp();
        // per-ray sum in sample order (k_sum1), normalisation by clamp(sum, 1e-6), exclusive cumsum (k_cumsum<true>)
        float acc = 0.0f;
        for (int base = 0; base < rr.n; base += 32) {
            const int i = base + lane;
            const float v = (i < rr.n) ? cdf[rr.start + i] : 0.0f;
            const int cnt = min(32, rr.n - base);
            for (int k = 0; k < cnt; k++) acc = __fadd_rn(acc, __shfl_sync(kFull, v, k));
        }
        const float denom = fmaxf(acc, 1e-6f);
        float run = 0.0f;
        for (int base = 0; base < rr.n; base += 32) {
            const int i = base + lane;
            const float v = (i < rr.n) ? __fdiv_rn(cdf[rr.start + i], denom) : 0.0f;
            float mine = 0.0f;
            const int cnt = min(32, rr.n - base);
            for (int k = 0; k < cnt; k++) {
                const float vk = __shfl_sync(kFull, v, k);
                if (lane == k) mine = run;
                run = __fadd_rn(run, vk);
            }
            if (i < rr.n) cdf[rr.start + i] = mine;
        }
        __syncwarp();
    }
    // importance samples from the cdf (same body as k_importance_sample, one-sample rays included)
    const int ist = ray * nr_imp;
    const float ox = origins[3 * ray], oy = origins[3 * ray + 1], oz = origins[3 * ray + 2];
    const float dx = dirs[3 * ray], dy = dirs[3 * ray + 1], dz = dirs[3 * ray + 2];
    const float fixed_dt = ray_fixed_dt[ray];
    for (int i = lane; i < nr_imp; i += 32) {
        const int s = ist + i;
        if (skip || rr.n == 1) {
            o_pos[3 * s] = 0; o_pos[3 * s + 1] = 0; o_pos[3 * s + 2] = 0;
            o_dirs[3 * s] = 0; o_dirs[3 * s + 1] = 0; o_dirs[3 * s + 2] = 0;
            o_z[s] = -1.0f;
            continue;
        }
        const float du = (float)(1.0 / (double)(nr_imp + 1));
        float u = __fmaf_rn((float)i, du, du);
        if (jitter) {
            Pcg32 rng = rng0;
            rng.advance((int64_t)(i + 1) * (int64_t)ray + (int64_t)i);
            const float rnd = rng.next_float();
            const float mov = (float)((double)du / 2.0);
            u = __fadd_rn(u, map_range(rnd, 0.0f, 1.0f, -mov, mov));
        }
        u = clampf(u, (float)(0.0 + 1e-6), (float)(1.0 - 1e-5));
        const int imax = cdf_search(cdf, u, rr.start, rr.end - 1);
        const int imin = max(imax - 1, 0);
        const float cmax = cdf[imax], cmin = cdf[imin];
        const float zmax = z[imax], zmin = z[imin];
        float zi = map_range(u, cmin, cmax, zmin, zmax);
        float dmin = __fsub_rn(zi, zmin), dmax = __fsub_rn(zmax, zi);
        if (dmin < dmax) { dmin = fminf(dmin, fixed_dt); zi = __fadd_rn(zmin, dmin); }
        else { dmax = fminf(dmax, fixed_dt); zi = __fsub_rn(zmax, dmax); }
        o_pos[3 * s] = __fmaf_rn(zi, dx, ox); o_pos[3 * s + 1] = __fmaf_rn(zi, dy, oy); o_pos[3 * s + 2] = __fmaf_rn(zi, dz, oz);
        o_dirs[3 * s] = dx; o_dirs[3 * s + 1] = dy; o_dirs[3 * s + 2] = dz;
        o_z[s] = zi;
    }
}

// VolumeRenderingGPU.cuh:950-1131. Two-pointer merge of the uniform and importance samples of one ray.
// Lane 0 replays the reference's merge decisions into shared memory (source index per output slot), then
// the whole warp materialises positions / dirs / z / sdf / dt with coalesced stores. Output slots come from
// an exclusive scan (offsets) instead of an atomic counter. A ray longer than the shared-memory stage is merged
// by lane 0 alone, straight from and to global memory, with the same decisions and arithmetic.
constexpr int kMergeCap = 1024;  // max merged samples per ray handled in shared memory
__global__ void __launch_bounds__(128)
k_combine(int nr_rays, const float* __restrict__ origins, const float* __restrict__ dirs, const float* __restrict__ t_exit_,
          const int* __restrict__ u_start_end, const float* __restrict__ u_fixed_dt, bool equal, int fixed_n,
          const float* __restrict__ u_z, const float* __restrict__ u_sdf, bool u_has_sdf, int imp_n,
          const float* __restrict__ i_z, const float* __restrict__ i_sdf, bool i_has_sdf, int c_max,
          const int* __restrict__ offsets, const int* __restrict__ block_sums, int scan_block, float* __restrict__ c_pos,
          float* __restrict__ c_dirs, float* __restrict__ c_z, float* __restrict__ c_dt, float* __restrict__ c_sdf,
          float* __restrict__ c_fixed_dt, int* __restrict__ c_start_end) {
    __shared__ float zs[4][kMergeCap];
    __shared__ short src[4][kMergeCap];
    int wib = threadIdx.x >> 5;
    int ray = blockIdx.x * 4 + wib;
    int lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    RayRange ur = ray_range(ray, u_start_end, equal, fixed_n);
    if (ur.n <= 1) {
        if (lane == 0) { c_fixed_dt[ray] = 0; reinterpret_cast<int2*>(c_start_end)[ray] = make_int2(0, 0); }
        return;
    }
    int cn = ur.n + imp_n;
    int cs = offsets[ray] + block_sums[ray / scan_block];
    if (lane == 0) reinterpret_cast<int2*>(c_start_end)[ray] = make_int2(cs, cs + cn);
    if (cs + cn > c_max) return;
    float fixed_dt = u_fixed_dt[ray];
    if (lane == 0) c_fixed_dt[ray] = fixed_dt;
    int ist = ray * imp_n;
    if (cn > kMergeCap) {
        if (lane != 0) return;
        float ox = origins[3 * ray], oy = origins[3 * ray + 1], oz = origins[3 * ray + 2];
        float dx = dirs[3 * ray], dy = dirs[3 * ray + 1], dz = dirs[3 * ray + 2];
        int iu = 0, ii = 0;
        float prev = 0.0f;
        for (int i = 0; i < cn; i++) {
            float zu = (iu < ur.n) ? u_z[ur.start + iu] : 1e10f;
            float zi = (ii < imp_n) ? i_z[ist + ii] : 1e10f;
            bool take_u = zu < zi;
            float zz = take_u ? zu : zi;
            int s = cs + i;
            c_pos[3 * s] = __fmaf_rn(zz, dx, ox); c_pos[3 * s + 1] = __fmaf_rn(zz, dy, oy); c_pos[3 * s + 2] = __fmaf_rn(zz, dz, oz);
            c_dirs[3 * s] = dx; c_dirs[3 * s + 1] = dy; c_dirs[3 * s + 2] = dz;
            c_z[s] = zz;
            if (take_u) { if (u_has_sdf) c_sdf[s] = u_sdf[ur.start + iu]; iu++; }
            else { if (i_has_sdf) c_sdf[s] = i_sdf[ist + ii]; ii++; }
            if (i > 0) c_dt[s - 1] = fminf(__fsub_rn(zz, prev), fixed_dt);
            prev = zz;
        }
        c_dt[cs + cn - 1] = clampf(__fsub_rn(t_exit_[ray], prev), 0.0f, fixed_dt);
        return;
    }
    // stage both z lists: uniform at [0,n), importance at [n, n+imp)
    for (int i = lane; i < ur.n; i += 32) zs[wib][i] = u_z[ur.start + i];
    for (int i = lane; i < imp_n; i += 32) zs[wib][ur.n + i] = i_z[ist + i];
    __syncwarp();
    if (lane == 0) {
        int iu = 0, ii = 0;
        for (int i = 0; i < cn; i++) {
            float zu = (iu < ur.n) ? zs[wib][iu] : 1e10f;
            float zi = (ii < imp_n) ? zs[wib][ur.n + ii] : 1e10f;
            if (zu < zi) { src[wib][i] = (short)iu; iu++; }
            else { src[wib][i] = (short)(ur.n + ii); ii++; }   // note: may read past imp_n only when both exhausted (never: i<cn)
        }
    }
    __syncwarp();
    float ox = origins[3 * ray], oy = origins[3 * ray + 1], oz = origins[3 * ray + 2];
    float dx = dirs[3 * ray], dy = dirs[3 * ray + 1], dz = dirs[3 * ray + 2];
    float t_exit = t_exit_[ray];
    for (int i = lane; i < cn; i += 32) {
        int sidx = src[wib][i];
        float zz = zs[wib][sidx];
        int s = cs + i;
        c_pos[3 * s] = __fmaf_rn(zz, dx, ox); c_pos[3 * s + 1] = __fmaf_rn(zz, dy, oy); c_pos[3 * s + 2] = __fmaf_rn(zz, dz, oz);
        c_dirs[3 * s] = dx; c_dirs[3 * s + 1] = dy; c_dirs[3 * s + 2] = dz;
        c_z[s] = zz;
        if (sidx < ur.n) { if (u_has_sdf) c_sdf[s] = u_sdf[ur.start + sidx]; }
        else { if (i_has_sdf) c_sdf[s] = i_sdf[ist + sidx - ur.n]; }
        float dt;
        if (i < cn - 1) dt = fminf(__fsub_rn(zs[wib][src[wib][i + 1]], zz), fixed_dt);
        else dt = clampf(__fsub_rn(t_exit, zz), 0.0f, fixed_dt);
        c_dt[s] = dt;
    }
}
// per-ray output counts for k_combine: (n>1 ? n+imp_n : 0), block-local exclusive scan
constexpr int kScanThreads = 1024;
__global__ void __launch_bounds__(kScanThreads)
k_combine_counts(int nr_rays, const int* __restrict__ start_end, bool equal, int fixed_n, int imp_n,
                 int* __restrict__ offsets, int* __restrict__ block_sums) {
    __shared__ int sm[32];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int c = 0;
    if (i < nr_rays) { RayRange r = ray_range(i, start_end, equal, fixed_n); c = r.n > 1 ? r.n + imp_n : 0; }
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int v = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(kFull, v, o); if (lane >= o) v += t; }
    if (lane == 31) sm[w] = v;
    __syncthreads();
    if (w == 0) {
        int s = sm[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(kFull, s, o); if (lane >= o) s += t; }
        sm[lane] = s;
    }
    __syncthreads();
    if (w > 0) v += sm[w - 1];
    if (i < nr_rays) offsets[i] = v - c;
    if (threadIdx.x == blockDim.x - 1) block_sums[blockIdx.x] = v;
}
__global__ void __launch_bounds__(kScanThreads) k_scan_sums(int nblocks, int* __restrict__ block_sums, int* __restrict__ total) {
    // nblocks <= 1024 here (1M rays); serial carry over chunks otherwise
    __shared__ int sm[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += blockDim.x) {
        int i = base + threadIdx.x;
        int c = i < nblocks ? block_sums[i] : 0;
        int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        int v = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(kFull, v, o); if (lane >= o) v += t; }
        if (lane == 31) sm[w] = v;
        __syncthreads();
        if (w == 0) {
            int s = sm[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(kFull, s, o); if (lane >= o) s += t; }
            sm[lane] = s;
        }
        __syncthreads();
        if (w > 0) v += sm[w - 1];
        int cr = carry;
        if (i < nblocks) block_sums[i] = cr + v - c;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = cr + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

// VolumeRenderingGPU.cuh:1135-1205
__global__ void __launch_bounds__(kThreads)
k_cumprod_backward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
                   const float* __restrict__ g_bg, const float* __restrict__ alpha, const float* __restrict__ bg_T,
                   const float* __restrict__ cumsumLV, float* __restrict__ g_alpha) {
    RAY_PROLOGUE();
    if (skip) return;
    float gb = __fmul_rn(g_bg[ray], bg_T[ray]);
    for (int i = lane; i < rr.n; i += 32) {
        int s = rr.start + i;
        float ga = 0.0f;
        if (i < rr.n - 1) {
            float a = fmaxf(1e-6f, alpha[s]);
            ga = __fadd_rn(__fdiv_rn(cumsumLV[s + 1], a), __fdiv_rn(gb, a));
        }
        g_alpha[s] = ga;
    }
}
// VolumeRenderingGPU.cuh:1208-1269 ; reference_bug reproduces the green-for-blue read at :1247
__global__ void __launch_bounds__(kThreads)
k_integrate_backward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n,
                     const float* __restrict__ g_pred, const float* __restrict__ vals, const float* __restrict__ w,
                     bool reference_bug, float* __restrict__ g_vals, float* __restrict__ g_w) {
    RAY_PROLOGUE();
    if (skip) return;
    float gx = g_pred[3 * ray], gy = g_pred[3 * ray + 1], gz = g_pred[3 * ray + 2];
    for (int i = lane; i < rr.n; i += 32) {
        int s = rr.start + i;
        float c0 = vals[3 * s], c1 = vals[3 * s + 1], c2 = reference_bug ? c1 : vals[3 * s + 2];
        float ws = w[s];
        g_vals[3 * s] = __fmul_rn(gx, ws); g_vals[3 * s + 1] = __fmul_rn(gy, ws); g_vals[3 * s + 2] = __fmul_rn(gz, ws);
        g_w[s] = __fmaf_rn(gz, c2, __fmaf_rn(gx, c0, __fmul_rn(gy, c1)));   // reference SASS order
    }
}
// VolumeRenderingGPU.cuh:1271-1329
__global__ void __launch_bounds__(kThreads)
k_sum_backward(int nr_rays, int max_nr_samples, const int* __restrict__ start_end, bool equal, int fixed_n, int D,
               const float* __restrict__ g_ray, const float* __restrict__ g_sample, float* __restrict__ g_vals) {
    RAY_PROLOGUE();
    if (skip) return;
    for (int e = lane; e < rr.n * D; e += 32) {
        int v = e % D;
        size_t idx = (size_t)rr.start * D + e;
        g_vals[idx] = __fadd_rn(g_ray[ray * D + v], g_sample[idx]);
    }
}
// VolumeRenderingGPU.cuh:307-367
__global__ void __launch_bounds__(kThreads)
k_compute_dt(int nr_rays, bool use_t_exit, const float* __restrict__ t_exit, int max_nr_samples, const float* __restrict__ z,
             const int* __restrict__ start_end, bool equal, int fixed_n, float* __restrict__ dt) {
    RAY_PROLOGUE();
    if (skip) return;
    for (int i = lane; i < rr.n; i += 32) {
        int s = rr.start + i;
        float next = (i < rr.n - 1) ? z[s + 1] : (use_t_exit ? t_exit[ray] : 1e10f);
        dt[s] = __fsub_rn(next, z[s]);
    }
}
// VolumeRenderingGPU.cuh:68-155 ; fused NeRF compositing with the T<1e-4 early out
__global__ void __launch_bounds__(kThreads)
k_render_nerf(int nr_rays, const float* __restrict__ rgb, const float* __restrict__ radiance, int max_nr_samples,
              const float* __restrict__ z, const float* __restrict__ dt_, const int* __restrict__ start_end, bool equal,
              int fixed_n, float* __restrict__ pred_rgb, float* __restrict__ pred_depth, float* __restrict__ bg_T,
              float* __restrict__ w_out) {
    RAY_PROLOGUE();
    if (skip) {
        if (lane == 0) { pred_rgb[3 * ray] = 0; pred_rgb[3 * ray + 1] = 0; pred_rgb[3 * ray + 2] = 0; pred_depth[ray] = 0; bg_T[ray] = 1.0f; }
        return;
    }
    float T = 1.0f, ax = 0, ay = 0, az = 0, depth = 0;
    bool done = false;
    for (int base = 0; base < rr.n && !done; base += 32) {
        int i = base + lane;
        float al = 0, x = 0, y = 0, zz = 0, zd = 0;
        if (i < rr.n) {
            int s = rr.start + i;
            al = __fsub_rn(1.0f, __expf(__fmul_rn(-radiance[s], dt_[s])));
            x = rgb[3 * s]; y = rgb[3 * s + 1]; zz = rgb[3 * s + 2]; zd = z[s];
        }
        float myw = 0;
        bool wrote = false;
        int cnt = min(32, rr.n - base);
        for (int k = 0; k < cnt; k++) {
            if (T < 1e-4f) { done = true; break; }
            float ak = __shfl_sync(kFull, al, k);
            float wk = __fmul_rn(ak, T);
            ax = __fmaf_rn(wk, __shfl_sync(kFull, x, k), ax);
            ay = __fmaf_rn(wk, __shfl_sync(kFull, y, k), ay);
            az = __fmaf_rn(wk, __shfl_sync(kFull, zz, k), az);
            depth = __fmaf_rn(wk, __shfl_sync(kFull, zd, k), depth);
            T = __fmul_rn(T, __fsub_rn(1.0f, ak));
            if (lane == k) { myw = wk; wrote = true; }
        }
        if (wrote) w_out[rr.start + i] = myw;
    }
    if (lane == 0) { pred_rgb[3 * ray] = ax; pred_rgb[3 * ray + 1] = ay; pred_rgb[3 * ray + 2] = az; pred_depth[ray] = depth; bg_T[ray] = T; }
}
// VolumeRenderingGPU.cuh:158-303
__global__ void __launch_bounds__(kThreads)
k_render_nerf_backward(int nr_rays, const float* __restrict__ g_pred_rgb, const float* __restrict__ g_bg_T,
                       const float* __restrict__ pred_rgb, const float* __restrict__ bg_T, const float* __restrict__ rgb,
                       const float* __restrict__ radiance, int max_nr_samples, const float* __restrict__ dt_,
                       const int* __restrict__ start_end, bool equal, int fixed_n, float* __restrict__ g_rgb,
                       float* __restrict__ g_radiance) {
    RAY_PROLOGUE();
    if (skip) return;
    float gx = g_pred_rgb[3 * ray], gy = g_pred_rgb[3 * ray + 1], gz = g_pred_rgb[3 * ray + 2];
    float fx = pred_rgb[3 * ray], fy = pred_rgb[3 * ray + 1], fz = pred_rgb[3 * ray + 2];
    float gbg = g_bg_T[ray], lastT = bg_T[ray];
    float T = 1.0f, ux = 0, uy = 0, uz = 0;
    bool done = false;
    for (int base = 0; base < rr.n && !done; base += 32) {
        int i = base + lane;
        float al = 0, x = 0, y = 0, zz = 0, dt = 0;
        if (i < rr.n) {
            int s = rr.start + i;
            dt = dt_[s];
            al = __fsub_rn(1.0f, __expf(__fmul_rn(-radiance[s], dt)));
            x = rgb[3 * s]; y = rgb[3 * s + 1]; zz = rgb[3 * s + 2];
        }
        float myw = 0, mygrad = 0;
        bool wrote = false;
        int cnt = min(32, rr.n - base);
        for (int k = 0; k < cnt; k++) {
            if (T < 1e-4f) { done = true; break; }
            float ak = __shfl_sync(kFull, al, k);
            float xk = __shfl_sync(kFull, x, k), yk = __shfl_sync(kFull, y, k), zk = __shfl_sync(kFull, zz, k);
            float dtk = __shfl_sync(kFull, dt, k);
            float wk = __fmul_rn(ak, T);
            ux = __fmaf_rn(wk, xk, ux); uy = __fmaf_rn(wk, yk, uy); uz = __fmaf_rn(wk, zk, uz);
            T = __fmul_rn(T, __fsub_rn(1.0f, ak));
            float grad = 0;
            grad += gx * dtk * (T * xk - (fx - ux));
            grad += gy * dtk * (T * yk - (fy - uy));
            grad += gz * dtk * (T * zk - (fz - uz));
            grad += gbg * (-dtk * lastT);
            if (lane == k) { myw = wk; mygrad = grad; wrote = true; }
        }
        if (wrote) {
            int s = rr.start + i;
            g_rgb[3 * s] = gx * myw; g_rgb[3 * s + 1] = gy * myw; g_rgb[3 * s + 2] = gz * myw;
            g_radiance[s] = mygrad;
        }
    }
}

#define ST ((cudaStream_t)stream)
inline int ray_blocks(int nr_rays) { return div_up((long long)nr_rays * 32, kThreads); }
}  // namespace

extern "C" {
#define RSP_ARGS int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n
#define RSP_PASS nr_rays, max_nr_samples, ray_start_end, equal != 0, fixed_n
#define GUARD() if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG

int psdf_vr_cumprod_alpha2transmittance(RSP_ARGS, const float* one_minus_alpha, float* transmittance, float* bg_transmittance, void* stream) {
    GUARD();
    k_cumprod<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, one_minus_alpha, transmittance, bg_transmittance);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_integrate_with_weights(RSP_ARGS, const float* vals, const float* weights, float* out, void* stream) {
    GUARD();
    k_integrate<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, vals, weights, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_sdf2alpha(RSP_ARGS, const float* ray_fixed_dt, const float* samples_dt, const float* sdf, float inv_s, int dynamic_inv_s,
                      float inv_s_multiplier, float* alpha, void* stream) {
    GUARD();
    k_sdf2alpha<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, max_nr_samples, ray_start_end, ray_fixed_dt, samples_dt, equal != 0,
                                                         fixed_n, sdf, inv_s, dynamic_inv_s != 0, inv_s_multiplier, alpha);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_sum_over_each_ray(RSP_ARGS, int val_dim, const float* vals, float* sum_ray, float* sum_sample, void* stream) {
    GUARD();
    if (val_dim < 1 || val_dim > 32) return PSDF_ERR_UNSUPPORTED;
    if (val_dim == 1) k_sum1<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, vals, sum_ray, sum_sample);
    else k_sumD<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, val_dim, vals, sum_ray, sum_sample);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_cumsum_over_each_ray(RSP_ARGS, const float* vals, int inverse, float* out, void* stream) {
    GUARD();
    k_cumsum<false><<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, vals, inverse != 0, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_compute_cdf(RSP_ARGS, const float* weights, float* cdf, void* stream) {
    GUARD();
    k_cumsum<true><<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, weights, false, cdf);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_importance_sample(RSP_ARGS, const float* origins, const float* dirs, const float* ray_fixed_dt, const float* samples_z,
                              const float* cdf, int nr_imp, uint64_t rng_state, uint64_t rng_inc, int jitter, float* o_pos,
                              float* o_dirs, float* o_z, void* stream) {
    GUARD();
    k_importance_sample<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, origins, dirs, max_nr_samples, ray_start_end, ray_fixed_dt,
                                                                 equal != 0, fixed_n, samples_z, cdf, nr_imp,
                                                                 Pcg32(rng_state, rng_inc), jitter != 0, o_pos, o_dirs, o_z);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_importance_round(RSP_ARGS, const float* origins, const float* dirs, const float* ray_fixed_dt, const float* samples_dt,
                             const float* samples_z, const float* sdf, float inv_s, int dynamic_inv_s, float inv_s_multiplier, int nr_imp,
                             uint64_t rng_state, uint64_t rng_inc, int jitter, float* cdf, float* o_pos, float* o_dirs, float* o_z,
                             void* stream) {
    GUARD();
    k_importance_round<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, origins, dirs, max_nr_samples, ray_start_end, ray_fixed_dt, samples_dt,
                                                                equal != 0, fixed_n, samples_z, sdf, inv_s, dynamic_inv_s != 0,
                                                                inv_s_multiplier, nr_imp, Pcg32(rng_state, rng_inc), jitter != 0, cdf, o_pos,
                                                                o_dirs, o_z);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
long long psdf_vr_combine_workspace_bytes(int nr_rays) {
    int nblocks = div_up(nr_rays > 0 ? nr_rays : 1, kScanThreads);
    return (long long)sizeof(int) * ((long long)nr_rays + nblocks + 1);
}
// workspace: [offsets nr_rays][block_sums nblocks][total 1]; total (device) = number of merged samples written
int psdf_vr_combine_uniform_samples_with_imp(RSP_ARGS, const float* origins, const float* dirs, const float* t_exit,
                                             const float* u_fixed_dt, const float* u_z, const float* u_sdf, int u_has_sdf,
                                             int imp_n, const float* i_z, const float* i_sdf, int i_has_sdf, int c_max,
                                             int* workspace, float* c_pos, float* c_dirs, float* c_z, float* c_dt, float* c_sdf,
                                             float* c_fixed_dt, int* c_start_end, void* stream) {
    GUARD();
    (void)max_nr_samples;
    int nblocks = div_up(nr_rays, kScanThreads);
    int* offsets = workspace;
    int* block_sums = workspace + nr_rays;
    int* total = block_sums + nblocks;
    k_combine_counts<<<nblocks, kScanThreads, 0, ST>>>(nr_rays, ray_start_end, equal != 0, fixed_n, imp_n, offsets, block_sums);
    k_scan_sums<<<1, kScanThreads, 0, ST>>>(nblocks, block_sums, total);
    k_combine<<<div_up(nr_rays, 4), 128, 0, ST>>>(nr_rays, origins, dirs, t_exit, ray_start_end, u_fixed_dt, equal != 0, fixed_n, u_z,
                                                 u_sdf, u_has_sdf != 0, imp_n, i_z, i_sdf, i_has_sdf != 0, c_max, offsets,
                                                 block_sums, kScanThreads, c_pos, c_dirs, c_z, c_dt, c_sdf, c_fixed_dt,
                                                 c_start_end);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_cumprod_alpha2transmittance_backward(RSP_ARGS, const float* grad_bg_transmittance, const float* alpha,
                                                 const float* bg_transmittance, const float* cumsumLV, float* grad_alpha,
                                                 void* stream) {
    GUARD();
    k_cumprod_backward<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, grad_bg_transmittance, alpha, bg_transmittance, cumsumLV,
                                                                grad_alpha);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_integrate_with_weights_backward(RSP_ARGS, const float* grad_pred, const float* vals, const float* weights,
                                            int reference_bug, float* grad_vals, float* grad_weights, void* stream) {
    GUARD();
    k_integrate_backward<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, grad_pred, vals, weights, reference_bug != 0, grad_vals,
                                                                  grad_weights);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_sum_over_each_ray_backward(RSP_ARGS, int val_dim, const float* grad_sum_ray, const float* grad_sum_sample,
                                       float* grad_vals, void* stream) {
    GUARD();
    if (val_dim < 1 || val_dim > 32) return PSDF_ERR_UNSUPPORTED;
    k_sum_backward<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(RSP_PASS, val_dim, grad_sum_ray, grad_sum_sample, grad_vals);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_compute_dt(RSP_ARGS, int use_t_exit, const float* t_exit, const float* samples_z, float* dt, void* stream) {
    GUARD();
    k_compute_dt<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, use_t_exit != 0, t_exit, max_nr_samples, samples_z, ray_start_end,
                                                          equal != 0, fixed_n, dt);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_volume_render_nerf(RSP_ARGS, const float* rgb, const float* radiance, const float* samples_z, const float* samples_dt,
                               float* pred_rgb, float* pred_depth, float* bg_transmittance, float* weight_per_sample, void* stream) {
    GUARD();
    k_render_nerf<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, rgb, radiance, max_nr_samples, samples_z, samples_dt, ray_start_end,
                                                           equal != 0, fixed_n, pred_rgb, pred_depth, bg_transmittance,
                                                           weight_per_sample);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_vr_volume_render_nerf_backward(RSP_ARGS, const float* grad_pred_rgb, const float* grad_bg_transmittance,
                                        const float* pred_rgb, const float* bg_transmittance, const float* rgb,
                                        const float* radiance, const float* samples_dt, float* grad_rgb, float* grad_radiance,
                                        void* stream) {
    GUARD();
    k_render_nerf_backward<<<ray_blocks(nr_rays), kThreads, 0, ST>>>(nr_rays, grad_pred_rgb, grad_bg_transmittance, pred_rgb,
                                                                    bg_transmittance, rgb, radiance, max_nr_samples, samples_dt,
                                                                    ray_start_end, equal != 0, fixed_n, grad_rgb, grad_radiance);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
}  // extern "C"
