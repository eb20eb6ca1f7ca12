// SDF from an oriented point cloud (train_sdf_from_mesh.py:126-160) or from a point sequence (train_4d_sdf.py:200-222), sm_90a. Two kernels
// replace the per-op chains of one iteration:
//   k_surface_fit_points   the iteration's points: index_select of the cloud (points + normals) and AABB.rand_points_inside
//                          (aabb.py) from one uniform draw, into one contiguous [Ns + No, D] (D = 4: plus the box rows' time draw)  1 launch for ~8
//   k_surface_fit_loss     sdf_loss (sdf_utils.py:16-57, eik_clamp=None) over the Ns + No rows: the four means, the weighted total and
//                          the seeds d loss / d {sdf, grad} with torch's autograd conventions                                       1 for ~40
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
constexpr int kSlots = 4;                // sums of the loss kernel: eikonal (all rows), normal, |sdf| (surface), exp(-100 |sdf|) (box)
constexpr int kDetSlot = 7;              // DetBufs::loss [7, 11): this kernel's fixed-point sums
#define ST ((cudaStream_t)stream)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    return v;
}
__device__ __forceinline__ float sign_f(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }   // torch.sign (abs backward)

// ---------------------------------------------------------------------------------------------- points
struct PointsArgs {
    int P, Ns, No;
    const float* pts;              // [P,D]
    const float* nrm;              // [P,3]
    const long long* idx;          // [Ns]
    const float* u01;              // [No,3]
    float size[3], half[3], trans[3];
    float* x;                      // [Ns + No, D]: surface rows, then box rows
    float* n;                      // [Ns, 3]
    const float* ut;               // D = 4: [No] time column of the box rows
};
// Surface rows copy the drawn cloud rows (index_select); an index outside [0, P) gives a NaN row instead of reading out of bounds.
// Box rows: u * size - size / 2 + translation, each operation rounded on its own as torch does (no contraction into an FMA); at D = 4
// followed by the time draw ut (torch.cat([box, ut], 1)).
template <int D>
__global__ void __launch_bounds__(kThreads)
k_surface_fit_points(PointsArgs A) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < A.Ns) {
        const long long j = A.idx[i];
        const bool ok = j >= 0 && j < A.P;
#pragma unroll
        for (int k = 0; k < D; k++) {
            A.x[D * i + k] = ok ? A.pts[D * j + k] : __int_as_float(0x7fc00000);
            if (k < 3) A.n[3 * i + k] = ok ? A.nrm[3 * j + k] : __int_as_float(0x7fc00000);
        }
    } else if (i < A.Ns + A.No) {
        const int r = i - A.Ns;
#pragma unroll
        for (int k = 0; k < 3; k++)
            A.x[D * i + k] = __fadd_rn(__fsub_rn(__fmul_rn(A.u01[3 * r + k], A.size[k]), A.half[k]), A.trans[k]);
        if constexpr (D == 4) A.x[D * i + 3] = A.ut[r];
    }
}

// ---------------------------------------------------------------------------------------------- loss
struct LossArgs {
    unsigned long long* fx;        // deterministic mode: DetBufs::loss + kDetSlot (the four sums in fixed point), else NULL
    int Ns, No;
    const float* sdf;              // [Ns + No]
    const float* g;                // [Ns + No, 3] d sdf / dx
    const float* nrm;              // [Ns, 3] normals of the surface rows
    float w[kSlots];               // weights {eikonal, normal, sdf, off-surface}
    float c[kSlots];               // seed coefficients scale * w / count, count = {Ns + No, Ns, Ns, No}
    float scale;
    float* g_sdf;                  // [Ns + No]    (=)
    float* g_grad;                 // [Ns + No, 3] (=)
    float* acc;                    // [5] sums + ticket (zero on entry, left zero)
    float* loss;                   // [1]
    float* terms;                  // [4] unweighted means {eikonal, normal, sdf, off-surface}
};
// sdf_loss with eik_clamp=None, times scale:
//   eikonal  |‖g‖ - 1| over all rows; the norm backward is zero at ‖g‖ = 0, abs backward is sign (zero at ‖g‖ = 1)
//   normal   1 - cos(g, n) over the surface rows, F.cosine_similarity (eps 1e-8): <g / max(‖g‖, eps), n / max(‖n‖, eps)>. torch clamps the
//            norms in place without autograd, so the gradient still flows through ‖g‖: d cos / d g = m / c - g <g, m> / (‖g‖ c^2), c =
//            max(‖g‖, eps), m = n / max(‖n‖, eps), the second term zero at ‖g‖ = 0 (a zero gradient row gets -c_nrm m / eps)
//   sdf      |sdf| over the surface rows (seed zero at sdf = 0)
//   off      exp(-100 |sdf|) over the box rows (seed zero at sdf = 0)
__global__ void __launch_bounds__(kThreads)
k_surface_fit_loss(LossArgs A) {
    __shared__ float red[kSlots][kThreads / 32];
    __shared__ bool last;
    const int N = A.Ns + A.No;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float v[kSlots] = {0.f, 0.f, 0.f, 0.f};
    if (i < N) {
        const float gx = A.g[3 * i], gy = A.g[3 * i + 1], gz = A.g[3 * i + 2];
        const float gn = sqrtf(gx * gx + gy * gy + gz * gz);
        const float d = gn - 1.0f;
        v[0] = fabsf(d);
        const float ke = gn > 0.0f ? A.c[0] * sign_f(d) / gn : 0.0f;
        float Gx = ke * gx, Gy = ke * gy, Gz = ke * gz;
        const float s = A.sdf[i];
        if (i < A.Ns) {
            const float nx = A.nrm[3 * i], ny = A.nrm[3 * i + 1], nz = A.nrm[3 * i + 2];
            const float nn = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-8f);
            const float mx = nx / nn, my = ny / nn, mz = nz / nn;
            const float c = fmaxf(gn, 1e-8f);
            const float cs = gx / c * mx + gy / c * my + gz / c * mz;
            v[1] = 1.0f - cs;
            const float kc = -A.c[1] / c;
            const float kg = gn > 0.0f ? -A.c[1] * ((gx * mx + gy * my + gz * mz) / (gn * c * c)) : 0.0f;
            Gx += kc * mx - kg * gx; Gy += kc * my - kg * gy; Gz += kc * mz - kg * gz;
            v[2] = fabsf(s);
            A.g_sdf[i] = A.c[2] * sign_f(s);
        } else {
            const float e = expf(-100.0f * fabsf(s));
            v[3] = e;
            A.g_sdf[i] = A.c[3] * e * -100.0f * sign_f(s);
        }
        A.g_grad[3 * i] = Gx; A.g_grad[3 * i + 1] = Gy; A.g_grad[3 * i + 2] = Gz;
    }
#pragma unroll
    for (int q = 0; q < kSlots; q++) {
        const float t = warp_sum(v[q]);
        if (lane == 0) red[q][warp] = t;
    }
    __syncthreads();
    if (threadIdx.x < kSlots) {
        float t = 0.f;
        for (int w = 0; w < kThreads / 32; w++) t += red[threadIdx.x][w];
        if (t != 0.0f) {
            if (A.fx) fx_add(A.fx + threadIdx.x, t);
            else atomicAdd(A.acc + threadIdx.x, t);
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned t = atomicAdd(reinterpret_cast<unsigned*>(A.acc + kSlots), 1u);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!last || threadIdx.x != 0) return;
    __threadfence();
    float sums[kSlots];
    if (A.fx) {
        volatile unsigned long long* fx = A.fx;
        for (int q = 0; q < kSlots; q++) { sums[q] = (float)((double)(long long)fx[q] / kFxScale); fx[q] = 0ull; }
    } else {
        volatile float* acc = A.acc;
        for (int q = 0; q < kSlots; q++) sums[q] = acc[q];
    }
    const float t_eik = sums[0] / (float)N, t_nrm = sums[1] / (float)A.Ns, t_sdf = sums[2] / (float)A.Ns, t_off = sums[3] / (float)A.No;
    A.loss[0] = (t_eik * A.w[0] + t_nrm * A.w[1] + t_sdf * A.w[2] + t_off * A.w[3]) * A.scale;
    A.terms[0] = t_eik; A.terms[1] = t_nrm; A.terms[2] = t_sdf; A.terms[3] = t_off;
#pragma unroll
    for (int q = 0; q <= kSlots; q++) A.acc[q] = 0.0f;      // ticket (acc[4], as bits) included: ready for the next launch
}
PointsArgs points_args(int P, int Ns, int No, const float* pts, const float* nrm, const long long* idx, const float* u01,
                       const float box_size[3], const float box_translation[3], float* x, float* n) {
    PointsArgs A;
    A.P = P; A.Ns = Ns; A.No = No; A.pts = pts; A.nrm = nrm; A.idx = idx; A.u01 = u01; A.x = x; A.n = n; A.ut = nullptr;
    for (int k = 0; k < 3; k++) {
        A.size[k] = box_size[k];
        A.half[k] = box_size[k] / 2.0f;          // torch.as_tensor(size) / 2 in float32 (exact)
        A.trans[k] = box_translation[k];
    }
    return A;
}
}  // namespace

extern "C" {

// Points of one iteration, see k_surface_fit_points. Ns = 0 (no cloud: pts, nrm, idx and n may be NULL) gives AABB.rand_points_inside_u01.
int psdf_surface_fit_points(int P, int Ns, int No, const float* pts, const float* nrm, const long long* idx, const float* u01,
                            const float box_size[3], const float box_translation[3], float* x, float* n, void* stream) {
    if (Ns < 0 || No < 0 || P < 0 || !box_size || !box_translation || (Ns > 0 && (P < 1 || !pts || !nrm || !idx || !n)) || (No > 0 && !u01))
        return PSDF_ERR_ARG;
    const long long rows = (long long)Ns + No;
    if (rows * 3 > 0x7fffffffLL || (long long)P * 3 > 0x7fffffffLL) return PSDF_ERR_UNSUPPORTED;
    if (rows == 0) return PSDF_OK;
    if (!x) return PSDF_ERR_ARG;
    PointsArgs A = points_args(P, Ns, No, pts, nrm, idx, u01, box_size, box_translation, x, n);
    k_surface_fit_points<3><<<div_up((int)rows, kThreads), kThreads, 0, ST>>>(A);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// Points of one space-time iteration (train_4d_sdf.py:200-208), see k_surface_fit_points: cloud rows pts [P,4] (x, y, z, t), box rows from
// u01 [No,3] and the time draw ut [No,1].
int psdf_spacetime_fit_points(int P, int Ns, int No, const float* pts, const float* nrm, const long long* idx, const float* u01, const float* ut,
                              const float box_size[3], const float box_translation[3], float* x, float* n, void* stream) {
    if (Ns < 0 || No < 0 || P < 0 || !box_size || !box_translation || (Ns > 0 && (P < 1 || !pts || !nrm || !idx || !n)) ||
        (No > 0 && (!u01 || !ut)))
        return PSDF_ERR_ARG;
    const long long rows = (long long)Ns + No;
    if (rows * 4 > 0x7fffffffLL || (long long)P * 4 > 0x7fffffffLL) return PSDF_ERR_UNSUPPORTED;
    if (rows == 0) return PSDF_OK;
    if (!x) return PSDF_ERR_ARG;
    PointsArgs A = points_args(P, Ns, No, pts, nrm, idx, u01, box_size, box_translation, x, n);
    A.ut = ut;
    k_surface_fit_points<4><<<div_up((int)rows, kThreads), kThreads, 0, ST>>>(A);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// sdf_loss of one iteration in one launch, see k_surface_fit_loss. acc [5]: scratch, ZERO before the first call, left zero by every call.
int psdf_surface_fit_loss(int Ns, int No, const float* sdf, const float* grad, const float* nrm, float w_eik, float w_nrm, float w_sdf,
                          float w_off, float scale, float* g_sdf, float* g_grad, float* acc, float* loss, float* terms, void* stream) {
    if (Ns < 1 || No < 1 || !sdf || !grad || !nrm || !g_sdf || !g_grad || !acc || !loss || !terms) return PSDF_ERR_ARG;
    const long long rows = (long long)Ns + No;
    if (rows * 3 > 0x7fffffffLL) return PSDF_ERR_UNSUPPORTED;
    LossArgs A;
    const DetBufs* dbuf = det_buffers();
    A.fx = dbuf ? dbuf->loss + kDetSlot : nullptr;
    A.Ns = Ns; A.No = No; A.sdf = sdf; A.g = grad; A.nrm = nrm;
    A.w[0] = w_eik; A.w[1] = w_nrm; A.w[2] = w_sdf; A.w[3] = w_off;
    const double cnt[kSlots] = {(double)rows, (double)Ns, (double)Ns, (double)No};
    for (int q = 0; q < kSlots; q++) A.c[q] = (float)((double)scale * (double)A.w[q] / cnt[q]);
    A.scale = scale;
    A.g_sdf = g_sdf; A.g_grad = g_grad; A.acc = acc; A.loss = loss; A.terms = terms;
    k_surface_fit_loss<<<div_up((int)rows, kThreads), kThreads, 0, ST>>>(A);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
