// Shared device helpers for the PermutoSDF H100 hot path.
//
// Everything in this header is written from scratch for sm_90a. Where a helper mirrors a
// piece of reference arithmetic the reference location is cited so that parity can be audited:
//   Morton code / voxel <-> position : kernels/permuto_sdf/OccupancyGridGPU.cuh:37-71,112-193
//   DDA step                          : kernels/permuto_sdf/OccupancyGridGPU.cuh:95-109
//   pcg32                             : kernels/permuto_sdf/pcg32.h:45-171
//
// Floating point policy for the ray-path translation units (compiled with -fmad=false):
// every fused multiply-add is written explicitly with __fmaf_rn at exactly the places where
// nvcc 12.9 contracts the reference source (checked in the SASS of the reference
// kernels, see DESIGN.md "FMA map"), so integer decisions taken from floats (voxel index,
// sample counts) are bit-identical to the reference CUDA path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define PSDF_OK 0
#define PSDF_ERR_ARG -1
#define PSDF_ERR_LAUNCH -2
#define PSDF_ERR_UNSUPPORTED -3

#define PSDF_CHECK_LAUNCH()                                   \
    do {                                                      \
        cudaError_t e__ = cudaGetLastError();                 \
        if (e__ != cudaSuccess) return PSDF_ERR_LAUNCH;       \
    } while (0)

namespace psdf {

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------- pcg32 -------------------------------------
// 64-bit LCG state, XSH-RR output (pcg32.h:66-82), jump-ahead (pcg32.h:150-171).
struct Pcg32 {
    uint64_t state;
    uint64_t inc;
    static constexpr uint64_t kMult = 0x5851f42d4c957f2dULL;

    __host__ __device__ Pcg32() : state(0x853c49e6748fea9bULL), inc(0xda3e39cb94b95bdbULL) {}
    __host__ __device__ Pcg32(uint64_t s, uint64_t i) : state(s), inc(i) {}

    // device-resident generator (CUDA-graph replay): inc == 0 is not a valid pcg32 stream, it marks `state` as a device
    // pointer to {state, inc}; kernels call resolve() once before drawing
    __device__ __forceinline__ void resolve() {
        if (inc == 0) { const uint64_t* p = reinterpret_cast<const uint64_t*>(state); state = p[0]; inc = p[1]; }
    }
    __host__ __device__ __forceinline__ uint32_t next_uint() {
        uint64_t old = state;
        state = old * kMult + inc;
        uint32_t xs = (uint32_t)(((old >> 18u) ^ old) >> 27u);
        uint32_t rot = (uint32_t)(old >> 59u);
        return (xs >> rot) | (xs << ((~rot + 1u) & 31));
    }
    // uniform in [0,1): build a float in [1,2) from the top 23 bits and subtract 1 (pcg32.h:88-97)
    __host__ __device__ __forceinline__ float next_float() {
        uint32_t u = (next_uint() >> 9) | 0x3f800000u;
#ifdef __CUDA_ARCH__
        return __uint_as_float(u) - 1.0f;
#else
        union { uint32_t u; float f; } x; x.u = u; return x.f - 1.0f;
#endif
    }
    // advance by delta draws in O(log delta)
    __host__ __device__ __forceinline__ void advance(int64_t delta_) {
        uint64_t cur_mult = kMult, cur_plus = inc, acc_mult = 1u, acc_plus = 0u;
        uint64_t delta = (uint64_t)delta_;
        while (delta > 0) {
            if (delta & 1) { acc_mult *= cur_mult; acc_plus = acc_plus * cur_mult + cur_plus; }
            cur_plus = (cur_mult + 1) * cur_plus;
            cur_mult *= cur_mult;
            delta >>= 1;
        }
        state = acc_mult * state + acc_plus;
    }
};

// ---------------------------------------------------------------- Morton ------------------------------------
__host__ __device__ __forceinline__ uint32_t spread10(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
__host__ __device__ __forceinline__ uint32_t morton3(uint32_t x, uint32_t y, uint32_t z) {
    return spread10(x) | (spread10(y) << 1) | (spread10(z) << 2);
}
__host__ __device__ __forceinline__ uint32_t compact10(uint32_t x) {
    x &= 0x49249249u;
    x = (x | (x >> 2)) & 0xc30c30c3u;
    x = (x | (x >> 4)) & 0x0f00f00fu;
    x = (x | (x >> 8)) & 0xff0000ffu;
    x = (x | (x >> 16)) & 0x0000ffffu;
    return x;
}

struct GridGeom {
    int V;            // voxels per dim (power of two)
    float extent;     // world size of the cube
    float tx, ty, tz; // translation of the cube centre
    float inv_extent; // 1/extent when extent is a power of two (x/extent == x*inv exactly), else 0 -> IEEE division
    float inv_V;      // 1/V, exact: V is a power of two
};

#ifdef __CUDACC__
// world position -> linear Morton voxel index, as an int (can be >= V^3 or negative when outside).
// Reference op order (SASS of check_occupancy_gpu): sub, IEEE div, add .5, mul V, cvt.rzi.u32 (saturating).
__device__ __forceinline__ int pos_to_voxel(float px, float py, float pz, const GridGeom& g) {
    float Vf = (float)g.V;
    // division by a power of two is exact, so the multiply below is bit-identical to the reference's IEEE division
    float qx = __fsub_rn(px, g.tx), qy = __fsub_rn(py, g.ty), qz = __fsub_rn(pz, g.tz);
    if (g.inv_extent != 0.0f) { qx = __fmul_rn(qx, g.inv_extent); qy = __fmul_rn(qy, g.inv_extent); qz = __fmul_rn(qz, g.inv_extent); }
    else { qx = __fdiv_rn(qx, g.extent); qy = __fdiv_rn(qy, g.extent); qz = __fdiv_rn(qz, g.extent); }
    float x = __fmul_rn(__fadd_rn(qx, 0.5f), Vf);
    float y = __fmul_rn(__fadd_rn(qy, 0.5f), Vf);
    float z = __fmul_rn(__fadd_rn(qz, 0.5f), Vf);
    return (int)morton3(__float2uint_rz(x), __float2uint_rz(y), __float2uint_rz(z));
}

// compile-time choice between the exact reciprocal multiply (power-of-two extent) and the IEEE division, for marching loops
template <bool kInvMul>
__device__ __forceinline__ int pos_to_voxel_t(float px, float py, float pz, const GridGeom& g, float Vf) {
    float qx = __fsub_rn(px, g.tx), qy = __fsub_rn(py, g.ty), qz = __fsub_rn(pz, g.tz);
    if (kInvMul) { qx = __fmul_rn(qx, g.inv_extent); qy = __fmul_rn(qy, g.inv_extent); qz = __fmul_rn(qz, g.inv_extent); }
    else { qx = __fdiv_rn(qx, g.extent); qy = __fdiv_rn(qy, g.extent); qz = __fdiv_rn(qz, g.extent); }
    float x = __fmul_rn(__fadd_rn(qx, 0.5f), Vf);
    float y = __fmul_rn(__fadd_rn(qy, 0.5f), Vf);
    float z = __fmul_rn(__fadd_rn(qz, 0.5f), Vf);
    return (int)morton3(__float2uint_rz(x), __float2uint_rz(y), __float2uint_rz(z));
}

// voxel index -> centre (or corner) of the voxel in world space (OccupancyGridGPU.cuh:112-155).
// The reference mixes float and double literals; the float result of each step equals the
// correctly rounded float op for these constants except the half-voxel shift, which is done in
// double there (x + half_voxel with x float, half float -> float add), so plain float ops match.
__device__ __forceinline__ float3 voxel_to_pos(uint32_t idx, const GridGeom& g, bool centre) {
    float Vf = (float)g.V;
    float x = __fdiv_rn((float)compact10(idx), Vf);
    float y = __fdiv_rn((float)compact10(idx >> 1), Vf);
    float z = __fdiv_rn((float)compact10(idx >> 2), Vf);
    x = __fsub_rn(x, 0.5f); y = __fsub_rn(y, 0.5f); z = __fsub_rn(z, 0.5f);
    if (centre) {
        float half = (float)((double)(float)(1.0 / (double)g.V) / 2.0);
        x = __fadd_rn(x, half); y = __fadd_rn(y, half); z = __fadd_rn(z, half);
    }
    // x*extent + translation is contracted to one FFMA in the reference SASS
    x = __fmaf_rn(x, g.extent, g.tx);
    y = __fmaf_rn(y, g.extent, g.ty);
    z = __fmaf_rn(z, g.extent, g.tz);
    return make_float3(x, y, z);
}

__device__ __forceinline__ float safe_inv(float d) {
    return (fabs((double)d) < 1e-16) ? 0.0f : __frcp_rn(d);
}

// distance (in world units of a unit cube) to the next voxel boundary along the ray.
// Reference: floorf(p*V + .5 + .5*sign(d)) - p*V, both p*V contracted into FFMAs by nvcc.
__device__ __forceinline__ float dda_axis(float p, float d, float id, float Vf) {
    float s = d > 0.0f ? 0.5f : (d < 0.0f ? -0.5f : 0.0f);
    float a = __fadd_rn(__fmaf_rn(p, Vf, 0.5f), s);
    float fl = floorf(a);
    return __fmul_rn(__fmaf_rn(-p, Vf, fl), id);
}
__device__ __forceinline__ float dda_step(float px, float py, float pz, float dx, float dy, float dz,
                                          float ix, float iy, float iz, int V) {
    float Vf = (float)V;
    float tx = fabsf(dda_axis(px, dx, ix, Vf));
    float ty = fabsf(dda_axis(py, dy, iy, Vf));
    float tz = fabsf(dda_axis(pz, dz, iz, Vf));
    float t = fminf(fminf(tx, ty), tz);
    return fmaxf(__fmul_rn(t, 1.0f / Vf), 0.0f);   // V is a power of two: t / V == t * (1/V) exactly
}

// same step with the per-axis half-voxel signs (0.5 sign(d)) hoisted out of the march (they depend on the ray only)
__device__ __forceinline__ float dda_step_s(float px, float py, float pz, float sx, float sy, float sz, float ix, float iy, float iz,
                                            float Vf, float inv_V) {
    float tx = fabsf(__fmul_rn(__fmaf_rn(-px, Vf, floorf(__fadd_rn(__fmaf_rn(px, Vf, 0.5f), sx))), ix));
    float ty = fabsf(__fmul_rn(__fmaf_rn(-py, Vf, floorf(__fadd_rn(__fmaf_rn(py, Vf, 0.5f), sy))), iy));
    float tz = fabsf(__fmul_rn(__fmaf_rn(-pz, Vf, floorf(__fadd_rn(__fmaf_rn(pz, Vf, 0.5f), sz))), iz));
    return fmaxf(__fmul_rn(fminf(fminf(tx, ty), tz), inv_V), 0.0f);
}
__device__ __forceinline__ float half_sign(float d) { return d > 0.0f ? 0.5f : (d < 0.0f ? -0.5f : 0.0f); }

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fmaxf(lo, fminf(x, hi)); }

// march from (px,py,pz) along d until an occupied voxel is hit (position updated to the point inside it) or the grid is left
// (position updated to the exit point, returns false). Body of advance_sample_to_next_occupied_voxel
// (OccupancyGridGPU.cuh:817-895); shared by the stand-alone kernel and the fused sphere tracer. If the step budget V*sqrt(3) runs
// out the position stays where it was and the sample counts as inside, like the reference.
__device__ __forceinline__ bool occ_advance_to_next_occupied(const GridGeom& g, const uint8_t* __restrict__ occ, float& ox, float& oy, float& oz,
                                                            float dx, float dy, float dz) {
    const int nv = g.V * g.V * g.V;
    const float eps = 1e-6f;
    const float ix = safe_inv(dx), iy = safe_inv(dy), iz = safe_inv(dz);
    const double max_steps = (double)g.V * sqrt(3.0);
    float t = 0;
    int steps = 0;
    // The t recurrence does not depend on the occupancy bytes, so it runs kAhead steps ahead of them: each batch costs one load
    // latency instead of kAhead. Decisions are then taken in march order, exactly as one step at a time would.
    constexpr int kAhead = 8;
    while ((double)steps < max_steps) {
        float bx[kAhead], by[kAhead], bz[kAhead];
        int bv[kAhead];
        int m = 0;
        bool oob_at_m = false;
#pragma unroll
        for (int k = 0; k < kAhead; k++) {
            if (!oob_at_m && (double)(steps + k) < max_steps) {
                const float px = __fmaf_rn(dx, t, ox), py = __fmaf_rn(dy, t, oy), pz = __fmaf_rn(dz, t, oz);
                const int v = pos_to_voxel(px, py, pz, g);
                bx[k] = px; by[k] = py; bz[k] = pz; bv[k] = v;
                m = k + 1;
                if (v > (nv - 1) || v < 0) oob_at_m = true;        // this entry ends the march; nothing after it is needed
                else {
                    const float dn = dda_step(px, py, pz, dx, dy, dz, ix, iy, iz, g.V);
                    t = __fadd_rn(__fadd_rn(t, dn), eps);
                }
            }
        }
        uint8_t bo[kAhead];
#pragma unroll
        for (int k = 0; k < kAhead; k++) bo[k] = (k < m && !(oob_at_m && k == m - 1)) ? __ldg(occ + bv[k]) : 0;
#pragma unroll
        for (int k = 0; k < kAhead; k++) {
            if (k < m) {
                if (oob_at_m && k == m - 1) { ox = bx[k]; oy = by[k]; oz = bz[k]; return false; }
                if (bo[k]) { ox = bx[k]; oy = by[k]; oz = bz[k]; return true; }
            }
        }
        if (m == 0) break;
        steps += m;
    }
    return true;
}
// The same march as occ_advance_to_next_occupied, resumable: at most `max_batches` batches of 8 steps per call, the march state (t, steps)
// lives with the caller. Returns 0: still marching (call again with the same origin), 1: stopped inside the grid (occupied voxel
// reached, or step budget exhausted: position unchanged), 2: left the grid. On 1 / 2 the position is written like the one-shot version.
// Decisions are taken in the same order on the same values, so the result is bit-identical however the batches are cut.
__device__ __forceinline__ int occ_advance_resumable(const GridGeom& g, const uint8_t* __restrict__ occ, float& ox, float& oy, float& oz,
                                                     float dx, float dy, float dz, float& t, int& steps, int max_batches) {
    const int nv = g.V * g.V * g.V;
    const float eps = 1e-6f;
    const float ix = safe_inv(dx), iy = safe_inv(dy), iz = safe_inv(dz);
    const double max_steps = (double)g.V * sqrt(3.0);
    constexpr int kAhead = 8;
    for (int b = 0; b < max_batches; b++) {
        if (!((double)steps < max_steps)) return 1;
        float bx[kAhead], by[kAhead], bz[kAhead];
        int bv[kAhead];
        int m = 0;
        bool oob_at_m = false;
#pragma unroll
        for (int k = 0; k < kAhead; k++) {
            if (!oob_at_m && (double)(steps + k) < max_steps) {
                const float px = __fmaf_rn(dx, t, ox), py = __fmaf_rn(dy, t, oy), pz = __fmaf_rn(dz, t, oz);
                const int v = pos_to_voxel(px, py, pz, g);
                bx[k] = px; by[k] = py; bz[k] = pz; bv[k] = v;
                m = k + 1;
                if (v > (nv - 1) || v < 0) oob_at_m = true;
                else {
                    const float dn = dda_step(px, py, pz, dx, dy, dz, ix, iy, iz, g.V);
                    t = __fadd_rn(__fadd_rn(t, dn), eps);
                }
            }
        }
        uint8_t bo[kAhead];
#pragma unroll
        for (int k = 0; k < kAhead; k++) bo[k] = (k < m && !(oob_at_m && k == m - 1)) ? __ldg(occ + bv[k]) : 0;
#pragma unroll
        for (int k = 0; k < kAhead; k++) {
            if (k < m) {
                if (oob_at_m && k == m - 1) { ox = bx[k]; oy = by[k]; oz = bz[k]; return 2; }
                if (bo[k]) { ox = bx[k]; oy = by[k]; oz = bz[k]; return 1; }
            }
        }
        if (m == 0) return 1;
        steps += m;
    }
    return ((double)steps < max_steps) ? 0 : 1;
}
// one AdamW element update (math: optim.cu). The roundings are explicit so that every kernel applying it (optim.cu k_adamw / k_adamw_dp,
// iter_glue.cu k_adamw_multi) produces the same bits whatever the compiler would contract.
__device__ __forceinline__ void adamw_update(float& p, float& m, float& v, float g, float grad_scale, float decay, float step_size, float beta1,
                                             float beta2, float bias_c2_sqrt, float eps) {
    const float gr = __fmul_rn(g, grad_scale);
    const float pk = __fmul_rn(p, decay);
    m = __fmaf_rn(beta1, m, __fmul_rn(1.0f - beta1, gr));
    v = __fmaf_rn(beta2, v, __fmul_rn(__fmul_rn(1.0f - beta2, gr), gr));
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), bias_c2_sqrt), eps);
    p = __fmaf_rn(-step_size, __fdiv_rn(m, denom), pk);
}
// ---------------------------------------------------------------- deterministic mode (opt-in)
// Float atomics add in arrival order, so by default a gradient reduced over many threads differs from run to run in its last bits
// (and a training step amplifies that: Adam with eps 1e-15 makes a whole learning-rate step of a near-zero gradient, sampling
// decisions flip). psdf_set_deterministic(1, ...) switches the training path's reductions to 64-bit fixed point instead: every
// contribution is rounded to the grid 2^-34 (resolution 5.8e-11; contributions and totals up to +-5.3e8) and the integers are added,
// which is associative (and modular, so partial sums may wrap), so the totals are the same in every run; k_fx_flush then adds them to
// the float gradients (+=) and clears the accumulators. The accumulators are allocated when the mode is switched on.
constexpr double kFxScale = 17179869184.0;
__device__ __forceinline__ unsigned long long fx_of(float v) { return (unsigned long long)__double2ll_rn((double)v * kFxScale); }
__device__ __forceinline__ void fx_add(unsigned long long* acc, float v) { atomicAdd(acc, fx_of(v)); }
constexpr int kDetImages = 1 << 16;                 // calibration images with fixed-point gradients (later images: float atomics)
constexpr int kDetSdfW = 64 * 64, kDetRgbW = 128 * 128;
struct DetBufs {
    unsigned long long* sdf_lattice;   // [lattice_len]
    unsigned long long* sdf_mlp;       // [4 x kDetSdfW weights | 4 x 64 biases]
    unsigned long long* rgb_lattice;   // [lattice_len]
    unsigned long long* rgb_mlp;       // [4 x kDetRgbW weights | 4 x 128 biases]
    unsigned long long* neus;          // [3 kDetImages weight delta | 3 kDetImages bias | inv_s]
    unsigned long long* lip;           // [4]
    unsigned long long* loss;          // [14]: [0, 5) psdf_loss_terms, [5, 7) psdf_sphere_fit_loss, [7, 11) psdf_surface_fit_loss,
                                       //       [11, 13) psdf_nerf_loss_forward
    int* winner;                       // [voxels]: occupancy-update arbitration (rayops.cu)
    long long lattice_len, voxels;
};
const DetBufs* det_buffers();        // of the current device; nullptr when the mode is off (optim.cu)
constexpr int kFxMaxSegs = 12;
struct FxSegs {
    int n = 0;
    unsigned long long* src[kFxMaxSegs];
    float* dst[kFxMaxSegs];
    long long len[kFxMaxSegs];
    // accumulators src[0, len) -> destination dst[0, len); a destination entry is only touched where its accumulator is non-zero
    void add(unsigned long long* s, float* d, long long l) {
        if (d && l > 0 && n < kFxMaxSegs) { src[n] = s; dst[n] = d; len[n] = l; n++; }
    }
};
static __global__ void __launch_bounds__(256) k_fx_flush(FxSegs S) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (int s = 0; s < S.n; s++) {
        unsigned long long* __restrict__ src = S.src[s];
        float* __restrict__ dst = S.dst[s];
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S.len[s]; i += stride) {
            const unsigned long long v = src[i];
            if (v) { dst[i] += (float)((double)(long long)v / kFxScale); src[i] = 0ull; }
        }
    }
}
inline int fx_flush(const FxSegs& S, cudaStream_t stream) {
    long long m = 0;
    for (int s = 0; s < S.n; s++) m = S.len[s] > m ? S.len[s] : m;
    if (m == 0) return 0;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long blocks = (m + 255) / 256, cap = 8LL * sms;
    k_fx_flush<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, stream>>>(S);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
// one-time (per device and kernel) opt-in to more than 48 KB of dynamic shared memory; `slot` is a static array owned by the call site.
// The request is capped at what the device allows next to the kernel's static shared memory.
template <typename K>
inline void psdf_optin_smem(K kernel, int bytes, bool (&slot)[64]) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !slot[dev]) {
        int optin = bytes;
        cudaFuncAttributes fa;
        if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess &&
            cudaFuncGetAttributes(&fa, kernel) == cudaSuccess)
            bytes = min(bytes, optin - (int)fa.sharedSizeBytes);
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        if (dev >= 0 && dev < 64) slot[dev] = true;
    }
}
inline GridGeom make_grid_geom(int V, float extent, const float* t) {
    GridGeom g;
    g.V = V; g.extent = extent; g.tx = t[0]; g.ty = t[1]; g.tz = t[2];
    int ex = 0;
    float m = frexpf(extent, &ex);
    g.inv_extent = (m == 0.5f) ? 1.0f / extent : 0.0f;      // exact reciprocal only for powers of two
    g.inv_V = 1.0f / (float)V;
    return g;
}

// per-ray sample range, mirrors get_start_end_ray_indices (VolumeRenderingGPU.cuh:30-60)
struct RayRange { int start, end, n; };
__device__ __forceinline__ RayRange ray_range(int ray, const int* __restrict__ start_end, bool equal, int fixed_n) {
    RayRange r;
    if (equal) { r.start = ray * fixed_n; r.end = r.start + fixed_n; }
    else { int2 se = reinterpret_cast<const int2*>(start_end)[ray]; r.start = se.x; r.end = se.y; }
    r.n = r.end - r.start;
    return r;
}
#endif

} // namespace psdf
