// Fused permutohedral encoding + SDF MLP for sm_90a: positions in, {sdf, d sdf/d x, geometric feature} out;
// the 36..52 encoded features and every hidden activation stay on chip (registers -> shared memory operand
// tiles -> wgmma tensor cores -> accumulators -> registers). Replaces the reference's chain
//   permutohedral_encoding.forward -> 4x cuBLAS SGEMM + 3x GELU kernels (+ autograd.grad for the normal)
// of SDF.forward / SDF.get_sdf_and_gradient (permuto_sdf_py/models/models.py:176-259).
//
// Numerics. The reference runs the MLP in fp32 (TF32 explicitly off, train_permuto_sdf.py:65) and the parity
// bar is 1e-3 relative, so single-pass bf16/tf32 operands are not good enough for d sdf/d x. Every operand is
// split as x = hi + lo (two bf16, |x-hi-lo| <= 2^-17 |x|) and each product uses three wgmma
// (hi*hi + hi*lo + lo*hi, fp32 accumulation): ~1e-5 relative error at 3x the (tiny) MMA cost.
//
// The gradient is computed in forward mode: three tangent streams d/dx_j ride along the value stream through
// the same weights ( tz_l = W_l ta_{l-1}, ta_l = gelu'(z_l) * tz_l ), their level-0 input being d feat / d x_j,
// which is exact because barycentric weights are piecewise linear in x.
//
// Work mapping: the encoder threads of a sample row each compute some of its 16-byte operand cores (4 lattice levels = 8 features
// each) for all streams; wgmma products stay in the registers of the warpgroup that issues them, whose epilogue (bias, GELU / GELU',
// bf16 hi/lo split) writes the next layer's operand tiles from the fragments. Value only (k_sdf_fused, the sphere tracer): 128-sample
// tiles, 256 threads, two CTAs per SM (see value_rows). Value + tangents: two groups of 256 threads per CTA on 64-sample sub-tiles
// (k_sdf_fused_dual).
// Weights (hi+lo, pre-packed in the core-matrix operand layout by k_pack_mlp) are fetched once per CTA with one
// cp.async.bulk (TMA) and stay resident; CTAs are persistent over tiles.
#include "fused_common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf_fused;

namespace {
// Threads per CTA of the value-only kernels (inference forward, sphere tracer). They need 93 KB of shared memory: with 256 threads (2 per
// row, <= 128 registers) TWO CTAs share an SM, each on its own tile with its own barriers, so that one CTA's MMA / barrier / gather waits
// are filled by the other's work.
constexpr int kValueThreads = 256;
// Up to two independent sample sets per launch (the main samples and the off-surface points of a training iteration): each set starts on
// a tile boundary and has its own outputs (grad / geom may be NULL per set).
struct FwdSegs {
    int n[2];
    int tile0[3];
    const float* pos[2];
    float* sdf[2];
    float* grad[2];
    float* geom[2];
};
// directions of the three spatial tangents d / d x_j (concat_core)
__device__ constexpr float kUnit3[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};

// ---------------------------------------------------------------------------------------------- value-only layers in registers
// Layer l of a value-only 128-row tile (inference forward, sphere tracer): warpgroup mh forms rows 64 mh .. 64 mh + 63 of D = A W^T in
// its registers (umma::wg_mma_regs fragments) and consumes them itself -- bias + GELU into the next layer's operand cores, or the
// output values. No other warp reads or writes those rows of the operand tiles in between, so no CTA barrier separates the two.
// the fragment (32 floats, the first Np / 2 used) of rows 64 mh .. 64 mh + 63 of layer l
__device__ __forceinline__ void value_rows(float* acc, const MlpGeom& g, int l, int mh, const uint8_t* s_a, const uint8_t* s_blob) {
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = 0.f;
    const uint8_t *wh = s_blob + g.w_hi[l], *wl = s_blob + g.w_lo[l];
    const uint32_t ro = (uint32_t)(mh * 8 * kSBO_A);
    switch (g.Np[l] / 16) {
        case 1: streams_product<16, 1>(acc, s_a, 0, kATileBytes, ro, wh, wl, g.Kp[l], 0); break;
        case 2: streams_product<32, 1>(acc, s_a, 0, kATileBytes, ro, wh, wl, g.Kp[l], 0); break;
        case 3: streams_product<48, 1>(acc, s_a, 0, kATileBytes, ro, wh, wl, g.Kp[l], 0); break;
        default: streams_product<64, 1>(acc, s_a, 0, kATileBytes, ro, wh, wl, g.Kp[l], 0); break;
    }
}
// bias + GELU of a hidden layer's fragment -> the next layer's operand cores
__device__ __forceinline__ void gelu_to_tiles(const float* acc, const float* bias, int Np, int mh, uint8_t* s_a) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (8 * j < Np) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int c = frag_col(j);
                const float z0 = acc[4 * j + 2 * h] + bias[c], z1 = acc[4 * j + 2 * h + 1] + bias[c + 1];
                store_pair(s_a, s_a + kATileBytes, frag_row(mh, h), c, z0 * gelu_eval(z0).cdf, z1 * gelu_eval(z1).cdf);
            }
        }
    }
}

// Value only (sdf and geometric feature, no tangents). D = 3: positions [N,3]; D = 4: space-time positions [N,4] (x, y, z, t)
template <int D>
__global__ void __launch_bounds__(kValueThreads, 2)
k_sdf_fused(FusedParams P, FwdSegs G, const float2* __restrict__ lattice, const float* __restrict__ scale,
            const float* __restrict__ shift, const float* __restrict__ window, const uint8_t* __restrict__ blob) {
    constexpr int kGroups = kValueThreads / kTile;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_blob = smem;
    uint8_t* s_a = smem + P.g.total;                       // {hi, lo} x 16 KB
    LevelC* lc = reinterpret_cast<LevelC*>(s_a + 2 * kATileBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(lc + 1);  // [0] weights
    const int tid = threadIdx.x, warp = tid >> 5;
    const int row = tid & (kTile - 1), grp = tid >> 7;

    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_fence_init();
    }
    load_level_consts<D>(lc, P.L, scale, shift, window, tid, kValueThreads);
    __syncthreads();
    if (tid == 0) {
        umma::mbar_expect_tx(&bars[0], (uint32_t)P.g.total);
        umma::bulk_g2s(s_blob, blob, (uint32_t)P.g.total, &bars[0]);
    }
    umma::mbar_wait(&bars[0], 0);
    const int level_cores = P.L / 4;                        // 4 levels x 2 features = one 16-byte core row
    const int all_cores = P.g.Kp[0] / 8;

    const int ntiles = G.tile0[2];
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const bool seg1 = tile >= G.tile0[1];                         // every sample set starts on a tile boundary
        const int n = (tile - (seg1 ? G.tile0[1] : 0)) * kTile + row;   // row inside its set
        const bool valid = n < (seg1 ? G.n[1] : G.n[0]);
        const float* __restrict__ pos = seg1 ? G.pos[1] : G.pos[0];
        float* __restrict__ sdf_out = seg1 ? G.sdf[1] : G.sdf[0];
        float* __restrict__ geom_out = seg1 ? G.geom[1] : G.geom[0];
        float x[D];
#pragma unroll
        for (int i = 0; i < D; i++) x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;

        // ---------------- encoder: operand cores grp, grp + 2, ... of this row
        for (int kc = grp; kc < all_cores; kc += kGroups) {
            float fv[8];
            if (kc < level_cores) {
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    Simplex<D> s;
                    float2 v[D + 1];
                    const float2 a = level_features<D>(x, lc, kc * 4 + q, lattice, P.T, P.cap_mask, s, v);
                    fv[2 * q] = a.x; fv[2 * q + 1] = a.y;
                }
            } else {
                concat_core<0, D>(P, kc, x, nullptr, fv, nullptr);
            }
            store8(s_a, s_a + kATileBytes, row, kc, fv);
        }

        // ---------------- MLP: 4 dense layers on the tensor cores
#pragma unroll 1
        for (int l = 0; l < kNL; l++) {
            umma::fence_async_smem();
            __syncthreads();
            // warpgroup mh owns rows 64 mh .. 64 mh + 63 from the product to the outputs (see value_rows)
            const int mh = warp >> 2;
            float acc[32];
            value_rows(acc, P.g, l, mh, s_a, s_blob);
            const float* bias = reinterpret_cast<const float*>(s_blob + P.g.bias[l]);
            if (l < kNL - 1) {
                gelu_to_tiles(acc, bias, P.g.Np[l], mh, s_a);
            } else {
                const int nout = P.g.N[l], n0 = n - row, cnt = seg1 ? G.n[1] : G.n[0];
#pragma unroll
                for (int j = 0; j < 8; j++) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
#pragma unroll
                        for (int b = 0; b < 2; b++) {
                            const int c = frag_col(j) + b, nr = n0 + frag_row(mh, h);
                            if (c >= nout || nr >= cnt) continue;
                            const float v = acc[4 * j + 2 * h + b] + bias[c];
                            if (c == 0) sdf_out[nr] = v;
                            else if (geom_out) geom_out[(size_t)nr * (nout - 1) + c - 1] = v;
                        }
                    }
                }
            }
        }
        __syncthreads();   // all reads of this tile's operand tiles done before the next tile's encoder overwrites them
    }
}

// ---------------------------------------------------------------------------------------------- value + tangents, two groups per CTA
// A single CTA of 512 threads on 128-sample tiles would run its phases in lock step: all 16 warps gather, then all wait for the tensor
// core, then all run the epilogue. Two CTAs per SM would let one CTA's waits be filled by the other's work, but the operand tiles of
// four streams (128 KB) + the weight blob (57 KB) allow one. Here ONE CTA holds TWO independent groups of 256 threads, each working on
// its own 64-sample sub-tile (M = 64 MMAs, 64 KB of operand tiles, its own named barrier and 256 accumulator columns) and sharing the
// resident weights: the groups drift apart and each one's MMA / barrier / gather waits overlap the other's encoder and epilogue work.
// Warpgroup hc of a group forms columns 32 hc .. 32 hc + 31 of all four streams (M = 64, N = 32) and keeps them in registers: the
// m16n8 fragments are exactly what its epilogue consumes (every thread holds useful values), so these products never leave the SM;
// the next layer's operand cores are written as 4-byte bf16 pairs.
constexpr int kSub = 64;                        // samples per sub-tile
constexpr int kSubTileBytes = kSub * 64 * 2;    // one bf16 operand tile [64 x 64]
constexpr int kGroupThreads = 256;
constexpr int kStg = 69;                         // row stride (floats) of the output staging tile: 64 value columns max + 3 gradient columns

// D = 3: positions [N,3]; D = 4: space-time positions [N,4], whose three tangents are the spatial ones (d / d x, y, z)
template <int D>
__global__ void __launch_bounds__(2 * kGroupThreads, 1)
k_sdf_fused_dual(FusedParams P, FwdSegs G, const float2* __restrict__ lattice, const float* __restrict__ scale,
                 const float* __restrict__ shift, const float* __restrict__ window, const uint8_t* __restrict__ blob) {
    constexpr int S = 4;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_blob = smem;
    const int tid = threadIdx.x, warp = warp_uniform(tid >> 5), t = tid & 255;
    const int grp2 = warp >> 3;                                              // group of the CTA; t: thread inside the group
    uint8_t* s_a = smem + P.g.total + grp2 * (S * 2 * kSubTileBytes);       // this group's S streams x {hi, lo} x 8 KB
    LevelC* lc = reinterpret_cast<LevelC*>(smem + P.g.total + 2 * S * 2 * kSubTileBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(lc + 1);                    // [0] weights, [3] start skew
    const int lane = tid & 31;
    const int wg = warp & 7;                                                 // warp inside the group, 0..7
    const int row = t & (kSub - 1), eg = t >> 6;                             // encoder: 4 threads per sample row
    constexpr int kEnc = kGroupThreads / kSub;

    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_init(&bars[3], 1);
        umma::mbar_fence_init();
    }
    load_level_consts<D>(lc, P.L, scale, shift, window, tid, 2 * kGroupThreads);
    __syncthreads();
    if (tid == 0) {
        umma::mbar_expect_tx(&bars[0], (uint32_t)P.g.total);
        umma::bulk_g2s(s_blob, blob, (uint32_t)P.g.total, &bars[0]);
    }
    umma::mbar_wait(&bars[0], 0);
    const int level_cores = P.L / 4, all_cores = P.g.Kp[0] / 8;
    // epilogue mapping: warp quadrant q = rows 16 q .. 16 q + 15, column half hc = columns 32 hc .. 32 hc + 31 (the warpgroup's products)
    const int q = wg & 3, hc = wg >> 2;
    const int er0 = q * 16 + (lane >> 2);                                     // rows er0 and er0 + 8 of the sub-tile
    const int ec0 = hc * 32 + 2 * (lane & 3);                                 // columns ec0 + 8 j + {0, 1}

    const int nsub = G.tile0[2];                                             // in units of 64-sample sub-tiles (see launch_forward)
    // Two identical groups that start together stay in lock step (every unit is shared fairly), waiting for the tensor core at the same
    // time. Group 1 therefore starts half a sub-tile late: it waits until group 0 has finished the second layer of its first sub-tile;
    // from then on one group's MMA / accumulator-read phases meet the other's encoder / GELU / store phases.
    bool skew_pending = true;
    if (grp2 == 1 && blockIdx.x * 2 < nsub) { umma::mbar_wait(&bars[3], 0); skew_pending = false; }
    for (int sub = blockIdx.x * 2 + grp2; sub < nsub; sub += 2 * gridDim.x) {
        const bool seg1 = sub >= G.tile0[1];
        const int sub0 = seg1 ? G.tile0[1] : 0, nseg = seg1 ? G.n[1] : G.n[0];
        const float* __restrict__ pos = seg1 ? G.pos[1] : G.pos[0];
        float* __restrict__ sdf_out = seg1 ? G.sdf[1] : G.sdf[0];
        float* __restrict__ grad_out = seg1 ? G.grad[1] : G.grad[0];
        float* __restrict__ geom_out = seg1 ? G.geom[1] : G.geom[0];
        const int n = (sub - sub0) * kSub + row;
        const bool valid = n < nseg;
        float x[D];
#pragma unroll
        for (int i = 0; i < D; i++) x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;

        // ---------------- encoder: operand cores eg, eg + 4, ... of this row
        for (int kc = eg; kc < all_cores; kc += kEnc) {
            float fv[8], ft[3][8];
            if (kc < level_cores) {
#pragma unroll
                for (int qq = 0; qq < 4; qq++) {
                    const int l = kc * 4 + qq;
                    Simplex<D> s;
                    float2 v[D + 1], t[3];
                    const float2 a = level_features<D>(x, lc, l, lattice, P.T, P.cap_mask, s, v);
                    spatial_tangents<D>(s, v, lc->window[l], lc->scale + l * 4, t);
                    fv[2 * qq] = a.x; fv[2 * qq + 1] = a.y;
#pragma unroll
                    for (int j = 0; j < 3; j++) { ft[j][2 * qq] = t[j].x; ft[j][2 * qq + 1] = t[j].y; }
                }
            } else {
                concat_core<3, D>(P, kc, x, kUnit3, fv, ft);
            }
            store8(s_a, s_a + kSubTileBytes, row, kc, fv);
#pragma unroll
            for (int j = 0; j < 3; j++) store8(s_a + (1 + j) * 2 * kSubTileBytes, s_a + (1 + j) * 2 * kSubTileBytes + kSubTileBytes, row, kc, ft[j]);
        }

        // ---------------- MLP: 4 dense layers, M = 64
#pragma unroll 1
        for (int l = 0; l < kNL; l++) {
            umma::fence_async_smem();
            umma::bar_sync(1 + grp2, kGroupThreads);
            // acc[0] = z, acc[1 + j] = tz_j: this warpgroup's 32 (or, in a narrower output layer, 16) columns of the four streams
            float acc[S][16];
#pragma unroll
            for (int s = 0; s < S; s++)
#pragma unroll
                for (int i = 0; i < 16; i++) acc[s][i] = 0.f;
            const int ncols = min(32, P.g.Np[l] - hc * 32);
            if (ncols == 32) streams_product<32, S>(acc[0], s_a, 2 * kSubTileBytes, kSubTileBytes, 0, s_blob + P.g.w_hi[l], s_blob + P.g.w_lo[l], P.g.Kp[l], hc * 32);
            else if (ncols == 16) streams_product<16, S>(acc[0], s_a, 2 * kSubTileBytes, kSubTileBytes, 0, s_blob + P.g.w_hi[l], s_blob + P.g.w_lo[l], P.g.Kp[l], hc * 32);
            umma::bar_sync(1 + grp2, kGroupThreads);     // every product of the group has read this layer's operand tiles
            const float* bias = reinterpret_cast<const float*>(s_blob + P.g.bias[l]);
            const bool last = (l == kNL - 1);
            if (ncols > 0) {                              // this warp's columns exist in this layer (the output layer may be narrower)
                float* z = acc[0];
                float (*tz)[16] = acc + 1;
#pragma unroll
                for (int j = 0; j < 4; j++) {
#pragma unroll
                    for (int b = 0; b < 2; b++) {
                        const float bb = bias[ec0 + 8 * j + b];
                        z[4 * j + b] += bb; z[4 * j + 2 + b] += bb;
                    }
                }
                if (!last) {
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const GeluEval ge = gelu_eval(z[i]);
                        const float g1 = fmaf(z[i], ge.pdf, ge.cdf);
#pragma unroll
                        for (int j = 0; j < 3; j++) tz[j][i] *= g1;
                        z[i] *= ge.cdf;
                    }
#pragma unroll
                    for (int j = 0; j < 4; j++) {
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int r = er0 + 8 * h, c = ec0 + 8 * j, i = 4 * j + 2 * h;
                            store_pair(s_a, s_a + kSubTileBytes, r, c, z[i], z[i + 1]);
#pragma unroll
                            for (int k = 0; k < 3; k++) {
                                uint8_t* th = s_a + (1 + k) * 2 * kSubTileBytes;
                                store_pair(th, th + kSubTileBytes, r, c, tz[k][i], tz[k][i + 1]);
                            }
                        }
                    }
                    if (skew_pending && grp2 == 0 && l == 1) { if (t == 0) umma::mbar_arrive(&bars[3]); skew_pending = false; }
                } else {
                    // outputs are staged in shared memory (the operand tiles are dead: the last MMAs completed) and leave as whole rows:
                    // a fragment thread holds 2 columns of 2 rows, which would be 4-byte stores 128 bytes apart
                    const int nout = P.g.N[l];
                    float* stg = reinterpret_cast<float*>(s_a);            // [64][kStg]: sdf | geom (nout - 1) | grad (3)
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int r = er0 + 8 * h;
#pragma unroll
                        for (int j = 0; j < 4; j++) {
#pragma unroll
                            for (int b = 0; b < 2; b++) {
                                const int col = ec0 + 8 * j + b;
                                if (col < nout) stg[r * kStg + col] = z[4 * j + 2 * h + b];
                            }
                        }
                        if (hc == 0 && (lane & 3) == 0) { stg[r * kStg + 64] = tz[0][2 * h]; stg[r * kStg + 65] = tz[1][2 * h]; stg[r * kStg + 66] = tz[2][2 * h]; }
                    }
                }
            }
        }
        // ---------------- coalesced copy-out of the sub-tile's rows
        umma::bar_sync(1 + grp2, kGroupThreads);     // staging complete
        {
            const float* stg = reinterpret_cast<const float*>(s_a);
            const int nout = P.g.N[kNL - 1];
            const int n0 = (sub - sub0) * kSub;
            const int rows = min(kSub, nseg - n0);
            if (t < rows) sdf_out[n0 + t] = stg[t * kStg];
            if (grad_out) for (int i = t; i < rows * 3; i += kGroupThreads) grad_out[(size_t)n0 * 3 + i] = stg[(i / 3) * kStg + 64 + (i % 3)];
            if (geom_out) {
                const int gw = nout - 1;
                for (int i = t; i < rows * gw; i += kGroupThreads) geom_out[(size_t)n0 * gw + i] = stg[(i / gw) * kStg + 1 + (i % gw)];
            }
        }
        umma::bar_sync(1 + grp2, kGroupThreads);     // the staging area is the next sub-tile's operand tile
    }
}

// ---------------------------------------------------------------------------------------------- fused sphere tracing
// sphere_trace of the reference (permuto_sdf_py/utils/sdf_utils.py:120-218) is a Python loop: mask the unconverged rays, gather,
// evaluate the SDF network, step along the ray, advance to the next occupied voxel, scatter back -- ~12 launches and a host sync
// per iteration. Here one CTA owns 128 rays for the whole trace: positions and converged flags live in shared memory, each
// iteration is encoder -> 4 tensor-core layers -> step / occupancy advance, the weights stay resident, and a tile stops as soon
// as its 128 rays have converged. Per ray the arithmetic is the one of the loop (same network evaluation, p + (d * sdf) * mult in
// separate roundings, same DDA), so the traced points are bit-identical to it.
// Template on the network's input width D and the boundary primitive. D = 4 is the space-time SDF traced at one time value
// (train_4d_sdf.py:268, vis_4d_sdf.py:105: the loop concatenates a column filled with time_val before every model call); positions,
// directions, the step and the boundary test stay 3-D and only the encoder sees the fourth coordinate. BOX replaces the bounding-sphere
// test with AABB.check_point_inside_primitive (aabb.py:28-43). <3, false> is the original kernel.
struct TraceParams {
    int nr_iters;
    float sdf_mult, conv_thresh;
    int has_occ;            // 1: advance through the occupancy grid, 0: test against the bounding sphere
    psdf::GridGeom grid;
    float sph_radius, sph_cx, sph_cy, sph_cz;
};
// what the original kernel does not read: the time value (D = 4) and the box (BOX), as the fp32 values the reference compares against
// (p - t < max, p - t > min, min = -max). A separate, last kernel argument: the original kernel's arguments keep their offsets.
struct TraceExt {
    float time_val;
    float box_max[3], box_min[3], box_t[3];
};
template <int D, bool BOX>
__global__ void __launch_bounds__(kValueThreads, 2)
k_sdf_sphere_trace(FusedParams P, TraceParams Q, const float* __restrict__ pos_in, const float* __restrict__ dirs,
                   const float2* __restrict__ lattice, const float* __restrict__ scale, const float* __restrict__ shift,
                   const float* __restrict__ window, const uint8_t* __restrict__ blob, const uint8_t* __restrict__ occ,
                   float* __restrict__ pos_out, uint8_t* __restrict__ converged_out, int* __restrict__ queue, TraceExt X) {
    // Persistent CTAs over a global ray queue: a CTA owns 128 ray SLOTS; a slot whose ray has finished (converged, left the occupied
    // region, or used its nr_iters evaluations) writes its result and is refilled with the next unclaimed ray (one warp-aggregated
    // atomicAdd per warp and iteration), so every network evaluation runs on a full tile until the frame is drained. Per ray the
    // arithmetic is unchanged (results are stored by ray index), so the traced points stay bit-identical to the masked loop.
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_blob = smem;
    uint8_t* s_a = smem + P.g.total;                       // {hi, lo} x 16 KB
    LevelC* lc = reinterpret_cast<LevelC*>(s_a + 2 * kATileBytes);
    float* s_pos = reinterpret_cast<float*>(lc + 1);       // [128][3] current point of the slot's ray
    float* s_dir = s_pos + kTile * 3;                      // [128][3]
    int* s_ray = reinterpret_cast<int*>(s_dir + kTile * 3);   // [128] ray index of the slot, -1: empty
    int* s_it = s_ray + kTile;                             // [128] evaluations done for the slot's ray
    int* s_ms = s_it + kTile;                              // [128] DDA steps of a march in progress, -1: not marching
    float* s_mt = reinterpret_cast<float*>(s_ms + kTile);  // [128] march parameter t of a march in progress
    int* s_new = reinterpret_cast<int*>(s_mt + kTile);     // [128] |sdf| < threshold at the evaluation that started the march
    float* s_sdf = reinterpret_cast<float*>(s_new + kTile);   // [128] network output of the slot in this round
    int* s_flag = reinterpret_cast<int*>(s_sdf + kTile);   // [0]: queue drained
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_flag + 2);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row = tid & (kTile - 1), grp = tid >> 7;
    constexpr int kGroups = kValueThreads / kTile;
    if (tid == 0) {
        umma::mbar_init(&bars[0], 1);
        umma::mbar_fence_init();
        s_flag[0] = 0;
    }
    load_level_consts<D>(lc, P.L, scale, shift, window, tid, kValueThreads);
    __syncthreads();
    if (tid == 0) {
        umma::mbar_expect_tx(&bars[0], (uint32_t)P.g.total);
        umma::bulk_g2s(s_blob, blob, (uint32_t)P.g.total, &bars[0]);
    }
    // first assignment: CTA b starts with rays [128 b, 128 b + 128); the queue counter hands out the rays past 128 * gridDim.x
    if (grp == 0) {
        const int n = blockIdx.x * kTile + row;
        const bool ok = n < P.N;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            s_pos[row * 3 + i] = ok ? pos_in[(size_t)n * 3 + i] : 0.0f;
            s_dir[row * 3 + i] = ok ? dirs[(size_t)n * 3 + i] : 0.0f;
        }
        s_ray[row] = ok ? n : -1;
        s_it[row] = 0;
        s_ms[row] = -1;
    }
    __syncthreads();
    umma::mbar_wait(&bars[0], 0);
    const int level_cores = P.L / 4, all_cores = P.g.Kp[0] / 8;
    const float* bias3 = reinterpret_cast<const float*>(s_blob + P.g.bias[kNL - 1]);
    const int first_queued = gridDim.x * kTile;

    // A long empty-space march (hundreds of dependent DDA steps, ~25 us) must not stall the other 127 slots: the march after a step is
    // cut into rounds of kMarchBatches x 8 DDA steps; a slot whose march is not finished keeps its state (s_mt, s_ms) and sits out the
    // network evaluations until it is (occ_advance_resumable: same decisions in the same order, so the result does not change).
    constexpr int kMarchBatches = 8;
    int evaluations = 0;                                      // network evaluations of this CTA (same value in every thread)
    int rounds = 0, net_rounds = 0;
    while (true) {
        const bool occupied = s_ray[row] >= 0;
        const bool active = occupied && s_ms[row] < 0;       // evaluates the network in this round
        if (__syncthreads_count(occupied) == 0) break;       // no ray left in this tile (and the queue is drained)
        // the count is the same in every thread, but ptxas cannot prove so: the network evaluation below would be a divergent path
        // and its wgmma chains serialized (C7520)
        const int nact = warp_uniform(__syncthreads_count(active));
        evaluations += nact / kGroups;
        float x[D];
#pragma unroll
        for (int i = 0; i < 3; i++) x[i] = s_pos[row * 3 + i];
        if constexpr (D == 4) x[3] = X.time_val;
        const bool run_net = nact > 0 && Q.nr_iters > 0;      // uniform
        rounds++;
        net_rounds += run_net ? 1 : 0;
        if (active && run_net) {
            for (int kc = grp; kc < all_cores; kc += kGroups) {
                float fv[8];
                if (kc < level_cores) {
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        Simplex<D> s;
                        float2 v[D + 1];
                        const float2 a = level_features<D>(x, lc, kc * 4 + q, lattice, P.T, P.cap_mask, s, v);
                        fv[2 * q] = a.x; fv[2 * q + 1] = a.y;
                    }
                } else {
                    concat_core<0, D>(P, kc, x, nullptr, fv, nullptr);
                }
                store8(s_a, s_a + kATileBytes, row, kc, fv);
            }
        }
        float sdf = 0.f;
        if (run_net) {
#pragma unroll 1
            for (int l = 0; l < kNL; l++) {
                umma::fence_async_smem();
                __syncthreads();
                const int mh = warp >> 2;             // warpgroup mh owns rows 64 mh .. 64 mh + 63 (see value_rows)
                float acc[32];
                value_rows(acc, P.g, l, mh, s_a, s_blob);
                if (l < kNL - 1) {
                    gelu_to_tiles(acc, reinterpret_cast<const float*>(s_blob + P.g.bias[l]), P.g.Np[l], mh, s_a);
                } else if ((lane & 3) == 0) {         // column 0 of rows frag_row(mh, 0 / 1)
                    s_sdf[frag_row(mh, 0)] = acc[0] + bias3[0];
                    s_sdf[frag_row(mh, 1)] = acc[2] + bias3[0];
                }
            }
            __syncthreads();
            sdf = s_sdf[row];
        }
        // ---- step / march / refill: one thread per slot
        if (grp == 0) {
            bool need = !occupied && s_flag[0] == 0;           // empty slot: try the queue again unless it is known to be drained
            if (occupied) {
                const int ray = s_ray[row];
                const float dx = s_dir[row * 3], dy = s_dir[row * 3 + 1], dz = s_dir[row * 3 + 2];
                float px = x[0], py = x[1], pz = x[2];
                bool finished = true, conv = false, newly = false, within = true;
                float t = 0.f;
                int steps = 0;
                if (Q.nr_iters > 0) {
                    if (active) {                              // this round's evaluation: step along the ray
                        px = __fadd_rn(x[0], __fmul_rn(__fmul_rn(dx, sdf), Q.sdf_mult));
                        py = __fadd_rn(x[1], __fmul_rn(__fmul_rn(dy, sdf), Q.sdf_mult));
                        pz = __fadd_rn(x[2], __fmul_rn(__fmul_rn(dz, sdf), Q.sdf_mult));
                        newly = fabsf(sdf) < Q.conv_thresh;
                        s_it[row] = s_it[row] + 1;
                    } else {                                   // march in progress: origin = s_pos, state from the previous round
                        t = s_mt[row]; steps = s_ms[row]; newly = s_new[row] != 0;
                    }
                    if (Q.has_occ) {
                        const int st = psdf::occ_advance_resumable(Q.grid, occ, px, py, pz, dx, dy, dz, t, steps, kMarchBatches);
                        if (st == 0) {                         // not there yet: keep the march origin and state, sit out the next evaluation
                            finished = false;
                            if (active) { s_pos[row * 3] = px; s_pos[row * 3 + 1] = py; s_pos[row * 3 + 2] = pz; }
                            s_mt[row] = t; s_ms[row] = steps; s_new[row] = newly ? 1 : 0;
                        } else within = (st == 1);
                    } else if constexpr (BOX) {
                        const float q[3] = {__fsub_rn(px, X.box_t[0]), __fsub_rn(py, X.box_t[1]), __fsub_rn(pz, X.box_t[2])};
                        within = true;
#pragma unroll
                        for (int i = 0; i < 3; i++) within = within && q[i] < X.box_max[i] && q[i] > X.box_min[i];
                    } else {
                        const float qx = __fsub_rn(px, Q.sph_cx), qy = __fsub_rn(py, Q.sph_cy), qz = __fsub_rn(pz, Q.sph_cz);
                        within = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qy, qy)), __fmul_rn(qz, qz))) < Q.sph_radius;
                    }
                    if (finished) conv = newly || !within;
                }
                if (finished) {
                    s_ms[row] = -1;
                    if (conv || s_it[row] >= Q.nr_iters) {     // the ray is done: result out, slot free
                        pos_out[(size_t)ray * 3] = px; pos_out[(size_t)ray * 3 + 1] = py; pos_out[(size_t)ray * 3 + 2] = pz;
                        if (converged_out) converged_out[ray] = (uint8_t)conv;
                        need = true;
                    } else {
                        s_pos[row * 3] = px; s_pos[row * 3 + 1] = py; s_pos[row * 3 + 2] = pz;
                    }
                }
            }
            // refill: one atomicAdd per warp for all its free slots
            const unsigned want = __ballot_sync(0xffffffffu, need);
            if (want) {
                int base = 0;
                if (lane == __ffs(want) - 1) base = atomicAdd(queue, __popc(want));
                base = __shfl_sync(0xffffffffu, base, __ffs(want) - 1);
                if (need) {
                    const int nr = first_queued + base + __popc(want & ((1u << lane) - 1u));
                    if (nr < P.N) {
#pragma unroll
                        for (int i = 0; i < 3; i++) {
                            s_pos[row * 3 + i] = pos_in[(size_t)nr * 3 + i];
                            s_dir[row * 3 + i] = dirs[(size_t)nr * 3 + i];
                        }
                        s_ray[row] = nr;
                        s_it[row] = 0;
                        s_ms[row] = -1;
                    } else {
                        s_ray[row] = -1;
                        s_flag[0] = 1;
                    }
                }
            }
        }
        __syncthreads();      // slots of this round visible, accumulator reads done
    }
    __syncthreads();
    if (tid == 0 && evaluations) {      // statistics of the launch: network evaluations, rounds, rounds that ran the network, longest CTA
        atomicAdd(queue + 1, evaluations);
        atomicAdd(queue + 2, rounds);
        atomicAdd(queue + 3, net_rounds);
        atomicMax(queue + 4, rounds);
    }
}

#define ST ((cudaStream_t)stream)
}  // namespace

// the launch of k_sdf_sphere_trace<D, BOX> (psdf_sdf_sphere_trace, psdf_sdf_sphere_trace_dim)
template <int D, bool BOX>
static int launch_trace(const TraceExt& X, int N, int L, int T, const float* pos, const float* dirs, const float* lattice,
                        const float* scale_factor, const float* shift, const float* window, float points_scaling, int hidden, int out_dim,
                        const uint8_t* blob, int nr_iters, float sdf_multiplier, float sdf_converged_tresh, const uint8_t* occupancy, int V,
                        float extent, const float trans[3], float sphere_radius, const float sphere_center[3], float* pos_out,
                        uint8_t* converged, int* queue_counter, void* stream) {
    if (!queue_counter) return PSDF_ERR_ARG;
    if (N < 0 || L < 1 || L > kMaxLevels || (L % 4) != 0 || hidden > 64 || hidden % 16 != 0 || out_dim > 64 || nr_iters < 0)
        return PSDF_ERR_UNSUPPORTED;
    if (N == 0) return PSDF_OK;
    FusedParams P;
    P.N = N; P.L = L; P.T = T;
    P.cap_mask = t_magic(T);
    P.points_scaling = points_scaling;
    P.in_dim = (L + 2) * 2;
    if (P.in_dim > 64) return PSDF_ERR_UNSUPPORTED;
    P.g = make_geom(P.in_dim, hidden, out_dim);
    TraceParams Q;
    Q.nr_iters = nr_iters; Q.sdf_mult = sdf_multiplier; Q.conv_thresh = sdf_converged_tresh;
    Q.has_occ = occupancy ? 1 : 0;
    const float zero3[3] = {0.f, 0.f, 0.f};
    Q.grid = psdf::make_grid_geom(occupancy ? V : 1, occupancy ? extent : 1.0f, occupancy ? trans : zero3);
    Q.sph_radius = sphere_radius; Q.sph_cx = sphere_center[0]; Q.sph_cy = sphere_center[1]; Q.sph_cz = sphere_center[2];
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = (size_t)P.g.total + 2 * kATileBytes + sizeof(LevelC) + kTile * 12 * sizeof(float) + 80;
    { static bool optin_[64]; psdf::psdf_optin_smem(k_sdf_sphere_trace<D, BOX>, 227 * 1024, optin_); }
    const int ntiles = div_up(N, kTile);
    k_sdf_sphere_trace<D, BOX><<<min(min(ntiles, 2 * sms), 2 * kAccCtas), kValueThreads, smem, ST>>>(P, Q, pos, dirs, reinterpret_cast<const float2*>(lattice), scale_factor,
                                                                     shift, window, blob, occupancy, pos_out, converged, queue_counter, X);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

extern "C" {

int psdf_sdf_sphere_trace(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                          const float* shift, const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob,
                          int nr_iters, float sdf_multiplier, float sdf_converged_tresh, const uint8_t* occupancy, int V, float extent,
                          const float trans[3], float sphere_radius, const float sphere_center[3], float* pos_out, uint8_t* converged,
                          int* queue_counter, void* stream) {
    TraceExt X = {};
    return launch_trace<3, false>(X, N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, nr_iters,
                                  sdf_multiplier, sdf_converged_tresh, occupancy, V, extent, trans, sphere_radius, sphere_center, pos_out,
                                  converged, queue_counter, stream);
}

int psdf_sdf_sphere_trace_dim(int pos_dim, float time_val, int boundary_kind, const float boundary[6], int N, int L, int T, const float* pos,
                              const float* dirs, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                              float points_scaling, int hidden, int out_dim, const uint8_t* blob, int nr_iters, float sdf_multiplier,
                              float sdf_converged_tresh, const uint8_t* occupancy, int V, float extent, const float trans[3],
                              float* pos_out, uint8_t* converged, int* queue_counter, void* stream) {
    if ((pos_dim != 3 && pos_dim != 4) || (boundary_kind != 0 && boundary_kind != 1)) return PSDF_ERR_UNSUPPORTED;
    if (!boundary) return PSDF_ERR_ARG;
    TraceExt X = {};
    X.time_val = time_val;
    float radius = 0.f, center[3] = {0.f, 0.f, 0.f};
    if (boundary_kind == 0) {
        radius = boundary[0];
        for (int i = 0; i < 3; i++) center[i] = boundary[1 + i];
    } else {
        for (int i = 0; i < 3; i++) { X.box_max[i] = boundary[i]; X.box_min[i] = -boundary[i]; X.box_t[i] = boundary[3 + i]; }
    }
    auto launch = pos_dim == 3 ? (boundary_kind ? launch_trace<3, true> : launch_trace<3, false>)
                               : (boundary_kind ? launch_trace<4, true> : launch_trace<4, false>);
    return launch(X, N, L, T, pos, dirs, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, nr_iters, sdf_multiplier,
                  sdf_converged_tresh, occupancy, V, extent, trans, radius, center, pos_out, converged, queue_counter, stream);
}


long long psdf_sdf_mlp_blob_bytes(int in_dim, int hidden, int out_dim) {
    MlpGeom g = make_geom(in_dim, hidden, out_dim);
    return (long long)g.total + g.total_t;     // forward operands + transposed copy for the backward
}

int psdf_sdf_mlp_pack(int in_dim, int hidden, int out_dim, const float* W0, const float* b0, const float* W1, const float* b1,
                      const float* W2, const float* b2, const float* W3, const float* b3, uint8_t* blob, void* stream) {
    if (hidden > 64 || out_dim > 64 || in_dim > 64) return PSDF_ERR_UNSUPPORTED;
    MlpGeom g = make_geom(in_dim, hidden, out_dim);
    dim3 grid(div_up(64 * 64, 256), kNL);
    k_pack_mlp<<<grid, 256, 0, ST>>>(g, W0, b0, W1, b1, W2, b2, W3, b3, blob);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

// psdf_sdf_mlp_pack + the end-of-iteration counters in the same launch: step_dev [1] (int, AdamW step count) += 1 and it_dev [1] (float,
// iteration number) += 1 (either may be NULL)
int psdf_sdf_mlp_pack_advance(int in_dim, int hidden, int out_dim, const float* W0, const float* b0, const float* W1, const float* b1,
                              const float* W2, const float* b2, const float* W3, const float* b3, uint8_t* blob, int* step_dev, float* it_dev,
                              void* stream) {
    if (hidden > 64 || out_dim > 64 || in_dim > 64) return PSDF_ERR_UNSUPPORTED;
    MlpGeom g = make_geom(in_dim, hidden, out_dim);
    dim3 grid(div_up(64 * 64, 256), kNL);
    k_pack_mlp<<<grid, 256, 0, ST>>>(g, W0, b0, W1, b1, W2, b2, W3, b3, blob, step_dev, it_dev);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"

template <int D>
static int launch_forward(int L, int T, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                          float points_scaling, int hidden, int out_dim, const uint8_t* blob, int nseg, const int* Ns, const float* const* pos,
                          float* const* sdf, float* const* grad, float* const* geom, void* stream) {
    if (L < 1 || L > kMaxLevels || (L % 4) != 0 || hidden > 64 || hidden % 16 != 0 || out_dim > 64) return PSDF_ERR_UNSUPPORTED;
    FusedParams P;
    P.L = L; P.T = T;
    P.cap_mask = t_magic(T);
    P.points_scaling = points_scaling;
    P.in_dim = (L + 2) * 2;                       // D = 3 or 4, F = 2: E = 2 concat levels
    if (P.in_dim > 64) return PSDF_ERR_UNSUPPORTED;
    P.g = make_geom(P.in_dim, hidden, out_dim);
    FwdSegs G;
    int tiles = 0, total = 0;
    bool tangents = false;
    for (int i = 0; i < 2; i++) {
        const int n = i < nseg ? Ns[i] : 0;
        if (n < 0) return PSDF_ERR_ARG;
        G.n[i] = n; G.tile0[i] = tiles;
        G.pos[i] = n ? pos[i] : nullptr; G.sdf[i] = n ? sdf[i] : nullptr; G.grad[i] = n ? grad[i] : nullptr; G.geom[i] = n ? geom[i] : nullptr;
        if (n && (!pos[i] || !sdf[i])) return PSDF_ERR_ARG;
        tangents = tangents || (n && grad[i]);
        tiles += div_up(n, kTile);
        total += n;
    }
    G.tile0[2] = tiles;
    P.N = total;
    if (tiles == 0) return PSDF_OK;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const float2* lat = reinterpret_cast<const float2*>(lattice);
    if (tangents) {
        // value + tangents: two independent 64-sample groups per CTA
        FwdSegs H = G;
        int subs = 0;
        for (int i = 0; i < 2; i++) { H.tile0[i] = subs; subs += div_up(G.n[i], kSub); }
        H.tile0[2] = subs;
        size_t smem = (size_t)P.g.total + 2 * 4 * 2 * kSubTileBytes + sizeof(LevelC) + 64;
        { static bool optin_[64]; psdf::psdf_optin_smem(k_sdf_fused_dual<D>, 227 * 1024, optin_); }
        k_sdf_fused_dual<D><<<min(min(div_up(subs, 2), sms), kAccCtas), 2 * kGroupThreads, smem, ST>>>(P, H, lat, scale_factor, shift, window, blob);
    } else {
        size_t smem = (size_t)P.g.total + 2 * kATileBytes + sizeof(LevelC) + 64;
        { static bool optin_[64]; psdf::psdf_optin_smem(k_sdf_fused<D>, 113 * 1024, optin_); }
        k_sdf_fused<D><<<min(min(tiles, 2 * sms), 2 * kAccCtas), kValueThreads, smem, ST>>>(P, G, lat, scale_factor, shift, window, blob);
    }
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

extern "C" {

int psdf_sdf_fused_forward(int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor, const float* shift,
                           const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, float* sdf,
                           float* grad, float* geom, void* stream) {
    if (N < 0) return PSDF_ERR_UNSUPPORTED;
    return launch_forward<3>(L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, 1, &N, &pos, &sdf, &grad, &geom, stream);
}

// Two independent sample sets in ONE launch (the main samples of a training iteration and its off-surface points: 8 tiles more instead
// of a second, latency-bound launch of 8 CTAs). Value + tangent kernel when either set asks for its gradient.
int psdf_sdf_fused_forward_multi(int L, int T, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                                 float points_scaling, int hidden, int out_dim, const uint8_t* blob, int N0, const float* pos0, float* sdf0,
                                 float* grad0, float* geom0, int N1, const float* pos1, float* sdf1, float* grad1, float* geom1, void* stream) {
    const int Ns[2] = {N0, N1};
    const float* pos[2] = {pos0, pos1};
    float* sdf[2] = {sdf0, sdf1};
    float* grad[2] = {grad0, grad1};
    float* geom[2] = {geom0, geom1};
    return launch_forward<3>(L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, 2, Ns, pos, sdf, grad, geom, stream);
}

// psdf_sdf_fused_forward at either input width: pos [N, pos_dim], pos_dim 3 (psdf_sdf_fused_forward) or 4 (space-time positions; grad holds
// the three spatial derivatives).
int psdf_sdf_fused_forward_dim(int pos_dim, int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor,
                               const float* shift, const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob,
                               float* sdf, float* grad, float* geom, void* stream) {
    if (N < 0) return PSDF_ERR_UNSUPPORTED;
    if (pos_dim == 3)
        return launch_forward<3>(L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, 1, &N, &pos, &sdf, &grad, &geom, stream);
    if (pos_dim == 4)
        return launch_forward<4>(L, T, lattice, scale_factor, shift, window, points_scaling, hidden, out_dim, blob, 1, &N, &pos, &sdf, &grad, &geom, stream);
    return PSDF_ERR_UNSUPPORTED;
}


}  // extern "C"
