// Minimal hand-written wgmma / mbarrier / bulk-copy (TMA) primitives for sm_90a, inline PTX only (no CUTLASS). Used by the
// fused kernels for the dense layers of the small MLPs.
//
// Operand layout used everywhere: K-major, no-swizzle ("interleaved") canonical layout made of core matrices
// of 8 rows x 16 bytes stored as 128 contiguous bytes:
//     byte_offset(row, k) = (row / 8) * SBO + (k_bytes / 16) * LBO + (row % 8) * 16 + (k_bytes % 16)
// LBO = distance between core matrices adjacent along K, SBO = distance between 8-row groups along M/N. A tile in this
// layout read with the transpose flag is the MN-major operand of the product that reduces over its rows.
//
// Accumulators. wgmma leaves D in the registers of the issuing warpgroup (M = 64 rows per instruction): wg_mma_regs, for kernels
// whose epilogue consumes the fragments in place. Kernels that keep accumulators across phases (pre-activations reused by the
// backward sweep, weight gradients summed over all tiles of a CTA) or read them back in a per-row layout use wg_gemm, which stores
// every product to a per-CTA accumulator area [128 lanes][cols] fp32 in global memory (L2 resident: at most 256 KB per CTA),
// addressed like a tensor-memory address: taddr = (lane << 16) | column. Each kernel owns one static area (a __device__ array
// per device, sized for kAccCtas persistent CTAs), so launches of the same kernel must not run concurrently on one device.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- shared memory matrix descriptor (64 bit), no swizzle ------------------------------------------------------
// [0,14) start address >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [49,52) base offset = 0 | [62,64) swizzle = 0
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// ---- per-CTA accumulator area --------------------------------------------------------------------------------
struct AccArea { float* base; int cols; };
__device__ __forceinline__ AccArea& acc_area() { __shared__ AccArea a; return a; }
// thread 0 binds the CTA's area (`cols` fp32 columns per lane); a __syncthreads must follow before any access
__device__ __forceinline__ void acc_attach(float* base, int cols) { acc_area().base = base; acc_area().cols = cols; }
__device__ __forceinline__ float* acc_ptr(uint32_t lane, uint32_t col) {
    const AccArea a = acc_area();
    return a.base + (size_t)lane * a.cols + col;
}
// 32 lanes x 16 consecutive columns: thread t of the warp gets lane (base_lane + t)
__device__ __forceinline__ void tmem_ld16(uint32_t taddr, float* v) {
    const float4* p = reinterpret_cast<const float4*>(acc_ptr((taddr >> 16) + (threadIdx.x & 31), taddr & 0xffff));
#pragma unroll
    for (int i = 0; i < 4; i++) { const float4 q = p[i]; v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w; }
}
// 16 lanes x 32 consecutive columns in the layout of an M = 64 accumulator quadrant (rows 16q .. 16q+15 live in lanes
// 32q .. 32q+15): thread t of the warp gets, for j = 0..3, h = 0..1, b = 0..1,
//     v[4 j + 2 h + b] = lane (base_lane + t / 4 + 8 h), column (base_col + 8 j + 2 (t % 4) + b)
// i.e. the m16n8 accumulator fragment repeated over four 8-column blocks
__device__ __forceinline__ void tmem_ld16x32(uint32_t taddr, float* v) {
    const int t = threadIdx.x & 31;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const float* p = acc_ptr((taddr >> 16) + t / 4 + 8 * h, (taddr & 0xffff) + 2 * (t % 4));
#pragma unroll
        for (int j = 0; j < 4; j++) { const float2 q = *reinterpret_cast<const float2*>(p + 8 * j); v[4 * j + 2 * h] = q.x; v[4 * j + 2 * h + 1] = q.y; }
    }
}
// store counterpart of tmem_ld16
__device__ __forceinline__ void tmem_st16(uint32_t taddr, const float* v) {
    float4* p = reinterpret_cast<float4*>(acc_ptr((taddr >> 16) + (threadIdx.x & 31), taddr & 0xffff));
#pragma unroll
    for (int i = 0; i < 4; i++) p[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
}

// named barrier over a subset of the CTA's warps (ids 1..15; id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
// make generic-proxy shared-memory writes visible to the async proxy (tensor core / TMA reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma (bf16 x bf16 -> f32, D in registers, issued by a whole warpgroup) ---------------------------------------
// TA / TB: 0 = K-major operand, 1 = MN-major (transposed) operand
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n48(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, %28;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_n(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (N == 16) wgmma_n16<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 32) wgmma_n32<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 48) wgmma_n48<TA, TB>(d, a, b, scale_d);
    else wgmma_n64<TA, TB>(d, a, b, scale_d);
}

// Accumulator lane of fragment row r (0..63) of an M = 64 product: `m64` places it like an M = 64 tensor-memory accumulator
// (lane (r / 16) * 32 + r % 16, the other 16 lanes of each quadrant free for a second accumulator at lane offset 16),
// otherwise lane r (the caller's lane field selects rows 0..63 or 64..127 of an M = 128 accumulator).
__device__ __forceinline__ uint32_t frag_lane(int r, bool m64) { return m64 ? (uint32_t)(32 * (r >> 4) + (r & 15)) : (uint32_t)r; }

// The three split products D (+)= A_hi B_hi + A_hi B_lo + A_lo B_hi of one warpgroup's M = 64 x N block, D in its registers in the
// m16n8 fragment layout (warp w of the warpgroup, lane t: d[4 j + 2 h + b] = row 16 w + t / 4 + 8 h, column 8 j + 2 (t % 4) + b, the
// layout tmem_ld16x32 returns). Issue only: the caller brackets a batch with wgmma_fence() and wgmma_commit() + wgmma_wait0().
template <int N, int TA, int TB>
__device__ __forceinline__ void wg_mma_regs(float* d, uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl, uint32_t a_step, uint32_t b_step,
                                            int ksteps, bool accumulate) {
#pragma unroll 1
    for (int kk = 0; kk < ksteps; kk++) {
        const uint64_t oa = (uint64_t)kk * a_step, ob = (uint64_t)kk * b_step;
        wgmma_n<N, TA, TB>(d, ah + oa, bh + ob, (kk > 0 || accumulate) ? 1u : 0u);
        wgmma_n<N, TA, TB>(d, ah + oa, bl + ob, 1u);
        wgmma_n<N, TA, TB>(d, al + oa, bh + ob, 1u);
    }
}

// S independent chains of wg_mma_regs sharing the B operand (stream s: A descriptors ah[s] / al[s], D = d + 16 s), in ONE k-step loop:
// k-step kk issues the three split products of every stream. Each stream's products accumulate in the order wg_mma_regs gives them.
// One loop rather than S loops one after the other: ptxas serializes the chains of S guarded loops (a wait after every HGMMA).
template <int N, int TA, int TB, int S>
__device__ __forceinline__ void wg_mma_streams(float* d, const uint64_t* ah, const uint64_t* al, uint64_t bh, uint64_t bl, uint32_t a_step,
                                               uint32_t b_step, int ksteps, bool accumulate) {
    if constexpr (S == 1) {
        wg_mma_regs<N, TA, TB>(d, ah[0], al[0], bh, bl, a_step, b_step, ksteps, accumulate);
    } else {
#pragma unroll 1
        for (int kk = 0; kk < ksteps; kk++) {
            const uint64_t oa = (uint64_t)kk * a_step, ob = (uint64_t)kk * b_step;
#pragma unroll
            for (int s = 0; s < S; s++) {
                wgmma_n<N, TA, TB>(d + 16 * s, ah[s] + oa, bh + ob, (kk > 0 || accumulate) ? 1u : 0u);
                wgmma_n<N, TA, TB>(d + 16 * s, ah[s] + oa, bl + ob, 1u);
                wgmma_n<N, TA, TB>(d + 16 * s, al[s] + oa, bh + ob, 1u);
            }
        }
    }
}

template <int N, int TA, int TB>
__device__ __forceinline__ void wg_gemm_n(uint32_t tdst, bool m64, uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl, uint32_t a_step,
                                          uint32_t b_step, int ksteps, bool accumulate) {
    float d[N / 2];
    const int w = (threadIdx.x >> 5) & 3, t = threadIdx.x & 31;
    const uint32_t lane0 = tdst >> 16, col0 = (tdst & 0xffff) + 2 * (t % 4);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const float* p = acc_ptr(lane0 + frag_lane(16 * w + t / 4 + 8 * h, m64), col0);
#pragma unroll
        for (int j = 0; j < N / 8; j++) {
            float2 q = accumulate ? *reinterpret_cast<const float2*>(p + 8 * j) : make_float2(0.f, 0.f);
            d[4 * j + 2 * h] = q.x; d[4 * j + 2 * h + 1] = q.y;
        }
    }
    wgmma_fence();
    wg_mma_regs<N, TA, TB>(d, ah, al, bh, bl, a_step, b_step, ksteps, accumulate);
    wgmma_commit();
    wgmma_wait0();
#pragma unroll
    for (int h = 0; h < 2; h++) {
        float* p = acc_ptr(lane0 + frag_lane(16 * w + t / 4 + 8 * h, m64), col0);
#pragma unroll
        for (int j = 0; j < N / 8; j++) *reinterpret_cast<float2*>(p + 8 * j) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
    }
}

// One warpgroup (all 128 threads, warp-aligned) forms the three split products of an M = 64 x nn block,
//     D (+)= A_hi B_hi + A_hi B_lo + A_lo B_hi      (K = 16 ksteps, fp32 accumulation)
// and stores it to the accumulator columns [col(tdst), col(tdst) + nn). Descriptors address the block's origin; a_step / b_step
// advance them by one K16 step, b_n64 moves B by 64 columns (nn > 64 runs in 64-column pieces). nn % 16 == 0.
// Returns with the results stored; the caller orders them for other warps (barrier or mbarrier arrive).
template <int TA, int TB>
__device__ __forceinline__ void wg_gemm(uint32_t tdst, bool m64, uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl, uint32_t a_step,
                                        uint32_t b_step, uint32_t b_n64, int ksteps, int nn, bool accumulate) {
    for (int n0 = 0; n0 < nn; n0 += 64) {
        const uint64_t ob = (uint64_t)(n0 / 64) * b_n64;
        const uint32_t td = tdst + (uint32_t)n0;
        switch (min(nn - n0, 64) / 16) {
            case 1: wg_gemm_n<16, TA, TB>(td, m64, ah, al, bh + ob, bl + ob, a_step, b_step, ksteps, accumulate); break;
            case 2: wg_gemm_n<32, TA, TB>(td, m64, ah, al, bh + ob, bl + ob, a_step, b_step, ksteps, accumulate); break;
            case 3: wg_gemm_n<48, TA, TB>(td, m64, ah, al, bh + ob, bl + ob, a_step, b_step, ksteps, accumulate); break;
            default: wg_gemm_n<64, TA, TB>(td, m64, ah, al, bh + ob, bl + ob, a_step, b_step, ksteps, accumulate); break;
        }
    }
}

// ---- mbarrier ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
// 1-D bulk copy global -> shared through the TMA unit, completion on an mbarrier (bytes % 16 == 0)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// 1-D bulk copy shared -> global (TMA store). Bulk groups are per thread: the issuing thread commits and waits.
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }   // smem reusable
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }             // writes done

// split a float into bf16 hi + bf16 lo (x ~= hi + lo with ~2^-17 relative error)
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// two floats -> packed bf16x2 hi and lo words (x0 in the low half): 2 CVT.BF16X2 + 2 logic + 2 FADD
__device__ __forceinline__ void split2_bf16(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    float h0 = __uint_as_float(hi << 16), h1 = __uint_as_float(hi & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - h1), "f"(x0 - h0));
}
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

}  // namespace umma
