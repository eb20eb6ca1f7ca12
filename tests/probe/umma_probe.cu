// Hardware probes for the wgmma conventions the fused kernels rely on (test infrastructure, NOT part of the product library: built
// into tests/probe/libumma_probe.so, loaded only by tests/test_umma_probe_gpu.py and tests/test_fused_gpu.py).
//   mode 0: two M = 64 accumulators sharing the same columns, one at lane offset 0 and one at lane offset 16 (an M = 64 product is
//           stored to lanes (m / 16) * 32 + m % 16), both formed from MN-major operands (sample axis = MMA K dimension)
//   mode 1: D[128 x Kp] = A[128 x Np] * W[Np x Kp] with A K-major and B = the FORWARD weight tile ([Np rows][Kp] K-major along k)
//           consumed as an MN-major operand (reduction over the rows): the reverse GEMM without a transposed weight copy.
//   umma_probe_gemm / umma_probe_gemm_tn: self-tests of the descriptor conventions (K-major forward GEMM with the kernels' own split /
//           pack / load helpers; weight-gradient product with the sample axis as the MMA K dimension, MN-major operands).
#include "../../permuto_sdf_b200/csrc/fused_common.cuh"

using namespace psdf_fused;

namespace {
__device__ float g_acc_probe[kTile * 64];     // accumulator area of the single probe CTA

__device__ __forceinline__ void attach_and_fill(float value) {
    if (threadIdx.x == 0) umma::acc_attach(g_acc_probe, 64);
    __syncthreads();
    float z[16];
#pragma unroll
    for (int i = 0; i < 16; i++) z[i] = value;
    for (int c = 0; c < 4; c++) umma::tmem_st16(((uint32_t)((threadIdx.x >> 5) * 32) << 16) + c * 16, z);
    umma::fence_async_smem();
    __syncthreads();
}
__device__ __forceinline__ void dump_all(float* dump, int N) {
    __syncthreads();
    const int tid = threadIdx.x;
    for (int c = 0; c < 4; c++) {
        float z[16];
        umma::tmem_ld16(((uint32_t)((tid >> 5) * 32) << 16) + c * 16, z);
#pragma unroll
        for (int i = 0; i < 16; i++) if (c * 16 + i < N) dump[tid * N + c * 16 + i] = z[i];
    }
}
// dW-style product of two [128 x 64] tiles as MN-major operands into an M = 64 accumulator (one warpgroup)
__device__ __forceinline__ void gemm_tn(uint32_t tdst, const uint8_t* a_hi, const uint8_t* a_lo, const uint8_t* b_hi, const uint8_t* b_lo, int nn) {
    // MN-major, no swizzle: LBO = stride between 8-sample groups (K), SBO = stride between 8-column cores (MN)
    const uint64_t dah = umma::make_desc(umma::smem_u32(a_hi), kSBO_A, kLBO), dal = umma::make_desc(umma::smem_u32(a_lo), kSBO_A, kLBO);
    const uint64_t dbh = umma::make_desc(umma::smem_u32(b_hi), kSBO_A, kLBO), dbl = umma::make_desc(umma::smem_u32(b_lo), kSBO_A, kLBO);
    umma::wg_gemm<1, 1>(tdst, true, dah, dal, dbh, dbl, (2 * kSBO_A) >> 4, (2 * kSBO_A) >> 4, (8 * kLBO) >> 4, kTile / 16, nn, false);
}

__global__ void __launch_bounds__(kTile) k_probe(int mode, const float* __restrict__ A, const float* __restrict__ A2,
                                                const float* __restrict__ B, float* __restrict__ dump) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* a_hi = smem;
    uint8_t* a_lo = a_hi + kATileBytes;
    uint8_t* a2_hi = a_lo + kATileBytes;
    uint8_t* a2_lo = a2_hi + kATileBytes;
    uint8_t* b_hi = a2_lo + kATileBytes;
    uint8_t* b_lo = b_hi + kATileBytes;
    const int tid = threadIdx.x;
    // all three inputs are [128][64] row-major fp32, stored as K-major core-matrix tiles (row = tid)
    for (int kc = 0; kc < 8; kc++) {
        float va[8], va2[8], vb[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            va[i] = A[tid * 64 + kc * 8 + i];
            va2[i] = A2[tid * 64 + kc * 8 + i];
            vb[i] = B[tid * 64 + kc * 8 + i];
        }
        store8(a_hi, a_lo, tid, kc, va);
        store8(a2_hi, a2_lo, tid, kc, va2);
        store8(b_hi, b_lo, tid, kc, vb);
    }
    attach_and_fill(-7.0f);        // sentinel: lanes no product writes keep it
    if (mode == 0) {
        gemm_tn(0, a_hi, a_lo, b_hi, b_lo, 64);
        gemm_tn(16u << 16, a2_hi, a2_lo, b_hi, b_lo, 64);
    } else {
        // A = a tile [128 x 64] K-major; B = first 64 rows of the b tile = W[n = 0..63][k = 0..63], forward layout. Reduction index n:
        // 8-row groups of the weight tile are kSBO_A apart (K direction), the k cores kLBO (N direction)
        const uint64_t dbh = umma::make_desc(umma::smem_u32(b_hi), kSBO_A, kLBO), dbl = umma::make_desc(umma::smem_u32(b_lo), kSBO_A, kLBO);
        for (int mh = 0; mh < 2; mh++) {
            const uint32_t ao = (uint32_t)(mh * 8 * kSBO_A);
            const uint64_t dah = umma::make_desc(umma::smem_u32(a_hi) + ao, kLBO, kSBO_A), dal = umma::make_desc(umma::smem_u32(a_lo) + ao, kLBO, kSBO_A);
            umma::wg_gemm<0, 1>((uint32_t)(64 * mh) << 16, false, dah, dal, dbh, dbl, (2 * kLBO) >> 4, (2 * kSBO_A) >> 4, (8 * kLBO) >> 4, 4, 64,
                                false);
        }
    }
    dump_all(dump, 64);
}
// ---------------------------------------------------------------------------------------------- debug GEMM (descriptor check)
// rows [64 mh, 64 mh + 64) of D[128 x Np] = A[128 x Kp] W^T as the three split products (one warpgroup, see umma::wg_gemm). A tiles
// have the 8-row-group stride kSBO_A; the weight tile is [Np rows][Kp] K-major. Descriptor convention checked by
// tests/test_fused_gpu.py::test_umma_gemm_self_test: the first offset field (LBO) is the stride between core matrices adjacent along K,
// the second (SBO) between 8-row groups.
__device__ __forceinline__ void issue_gemm(uint32_t tmem_d, int mh, const uint8_t* a_hi, const uint8_t* a_lo, const uint8_t* w_hi,
                                           const uint8_t* w_lo, int Kp, int Np) {
    const uint32_t sbo_w = (Kp / 8) * kLBO;
    const uint32_t ao = (uint32_t)(mh * 8 * kSBO_A);
    const uint64_t dah = umma::make_desc(umma::smem_u32(a_hi) + ao, kLBO, kSBO_A), dal = umma::make_desc(umma::smem_u32(a_lo) + ao, kLBO, kSBO_A);
    const uint64_t dwh = umma::make_desc(umma::smem_u32(w_hi), kLBO, sbo_w), dwl = umma::make_desc(umma::smem_u32(w_lo), kLBO, sbo_w);
    umma::wg_gemm<0, 0>(tmem_d + ((uint32_t)(64 * mh) << 16), false, dah, dal, dwh, dwl, (2 * kLBO) >> 4, (2 * kLBO) >> 4, (8 * sbo_w) >> 4,
                        Kp / 16, Np, false);
}
// D[128 x N] = A[128 x K] * B[N x K]^T with the same split/pack/load helpers as the fused kernels.
__global__ void __launch_bounds__(kTile) k_debug_gemm(int N, int K, const float* __restrict__ A, const float* __restrict__ B,
                                                      float* __restrict__ D) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int Kp = pad16(K), Np = pad16(N);
    uint8_t* a_hi = smem;
    uint8_t* a_lo = a_hi + kATileBytes;
    uint8_t* w_hi = a_lo + kATileBytes;
    uint8_t* w_lo = w_hi + Np * Kp * 2;
    const int tid = threadIdx.x;
    for (int kc = 0; kc < Kp / 8; kc++) {
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { int k = kc * 8 + i; v[i] = k < K ? A[tid * K + k] : 0.f; }
        store8(a_hi, a_lo, tid, kc, v);
    }
    const int sbo = (Kp / 8) * kLBO;
    for (int e = tid; e < Np * Kp; e += kTile) {
        int n = e / Kp, k = e - n * Kp;
        float v = (n < N && k < K) ? B[n * K + k] : 0.f;
        __nv_bfloat16 hi, lo;
        umma::split_bf16(v, hi, lo);
        int off = (n / 8) * sbo + (k / 8) * kLBO + (n % 8) * 16 + (k % 8) * 2;
        *reinterpret_cast<__nv_bfloat16*>(w_hi + off) = hi;
        *reinterpret_cast<__nv_bfloat16*>(w_lo + off) = lo;
    }
    attach_and_fill(0.0f);
    for (int mh = 0; mh < 2; mh++) issue_gemm(0, mh, a_hi, a_lo, w_hi, w_lo, Kp, Np);
    dump_all(D, N);
}

// D[M x N] = A^T B over the 128 rows of two operand tiles (A [128 x M], B [128 x N], both stored like every activation tile:
// row = sample, 16-byte core rows along the columns), i.e. the weight-gradient product dW = zbar^T a with the sample axis as the
// MMA K dimension and both operands MN-major. `dump` receives all 128 accumulator lanes x 64 columns so that the lane of every
// accumulator row can be read off on the host.
__global__ void __launch_bounds__(kTile) k_debug_gemm_tn(int M, int N, const float* __restrict__ A, const float* __restrict__ B,
                                                         float* __restrict__ dump) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* a_hi = smem;
    uint8_t* a_lo = a_hi + kATileBytes;
    uint8_t* b_hi = a_lo + kATileBytes;
    uint8_t* b_lo = b_hi + kATileBytes;
    const int tid = threadIdx.x;
    for (int kc = 0; kc < 8; kc++) {
        float va[8], vb[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            int c = kc * 8 + i;
            va[i] = c < M ? A[tid * M + c] : 0.f;
            vb[i] = c < N ? B[tid * N + c] : 0.f;
        }
        store8(a_hi, a_lo, tid, kc, va);
        store8(b_hi, b_lo, tid, kc, vb);
    }
    attach_and_fill(0.0f);         // lanes the product does not write read back as zero
    gemm_tn(0, a_hi, a_lo, b_hi, b_lo, pad16(N));      // M = 64 product; rows past M are zero
    dump_all(dump, 64);
}

}  // namespace

extern "C" int umma_probe(int mode, const float* A, const float* A2, const float* B, float* dump, void* stream) {
    size_t smem = 6 * kATileBytes;
    cudaFuncSetAttribute(k_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_probe<<<1, kTile, smem, (cudaStream_t)stream>>>(mode, A, A2, B, dump);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int umma_probe_gemm_tn(int M, int N, const float* A, const float* B, float* dump, void* stream) {
    if (M < 1 || M > 64 || N < 1 || N > 64) return -2;
    int smem = 4 * kATileBytes;
    cudaFuncSetAttribute(k_debug_gemm_tn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    k_debug_gemm_tn<<<1, kTile, smem, (cudaStream_t)stream>>>(M, N, A, B, dump);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int umma_probe_gemm(int N, int K, const float* A, const float* B, float* D, void* stream) {
    if (N < 1 || N > 64 || K < 1 || K > 64) return -2;
    size_t smem = 2 * kATileBytes + 2 * (size_t)pad16(N) * pad16(K) * 2;
    cudaFuncSetAttribute(k_debug_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    k_debug_gemm<<<1, kTile, smem, (cudaStream_t)stream>>>(N, K, A, B, D);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
