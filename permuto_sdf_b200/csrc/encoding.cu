// Multi-resolution permutohedral-lattice hash encoding for sm_90a: forward (barycentric gather),
// backward to the lattice (warp-aggregated vector atomics), backward to positions, and the double
// backward needed by the eikonal / curvature losses.
//
// The algorithm is the one of the external `permutohedral_encoding` package the reference imports
// (permuto_sdf_py/models/models.py:20,149,186); its source is not vendored in the reference, the
// semantics implemented here are the published ones restated in SURVEY.md Appendix B:
// elevate (x+shift)*scale to the hyperplane, round to the remainder-0 lattice point, rank-sort the
// residuals, barycentric weights by rank, hash the D-int key of each of the D+1 simplex vertices
// (h = (h + key_i) * 2531011 over i, mod capacity), blend F features, multiply by the level window.
//
// Mapping. One thread per sample, all levels in that thread; a warp is 32 consecutive samples,
// i.e. neighbours on a ray, so on coarse levels the 32 lanes hit the same few 8-byte table rows (L1
// broadcast) and on fine levels each lane has 4*UNROLL independent gathers in flight against the
// L2-resident table (L*T*F*4 B = 33.5 MB at L=16 < 50 MB L2). Outputs are staged in shared memory
// and written as one contiguous [32, C] block per warp. The backward reduces duplicates inside the warp
// (match_any + segmented shuffle tree) before issuing one red.global.add.v2.f32 per distinct vertex.
// Position gradients need no atomics because a thread owns all levels of its sample.
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr unsigned kFull = 0xffffffffu;
constexpr int kEncThreads = 128;
constexpr int kGroups = kEncThreads / 32;   // level groups (warps) per block; a block covers 32 samples
constexpr int kMaxLevels = 32;

struct EncParams {
    int N, L, T, C;          // samples, levels, table capacity, output columns
    int concat;              // concat raw points
    float points_scaling;
    unsigned cap_mask;       // floor(2^32 / T): multiplier of the division-free h mod T (see vertex_index)
};

template <int D>
struct Simplex {
    int rem0[D + 1];
    int rank[D + 1];
    float bary[D + 2];
};

// elevation of a D-vector of (already scaled) coordinates to the (D+1)-dim hyperplane
template <int D>
__device__ __forceinline__ void elevate(const float* cf, float* elevated) {
    float sm = 0.0f;
#pragma unroll
    for (int i = D; i > 0; i--) {
        elevated[i] = __fmaf_rn(-(float)i, cf[i - 1], sm);
        sm = __fadd_rn(sm, cf[i - 1]);
    }
    elevated[0] = sm;
}

// locate the enclosing simplex: remainder-0 point, rank permutation and barycentric weights
template <int D>
__device__ __forceinline__ void locate(const float* elevated, Simplex<D>& s) {
    const float inv = 1.0f / (float)(D + 1);
    int sum = 0;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float v = __fmul_rn(elevated[i], inv);
        float up = __fmul_rn(ceilf(v), (float)(D + 1));
        float down = __fmul_rn(floorf(v), (float)(D + 1));
        s.rem0[i] = (__fsub_rn(up, elevated[i]) < __fsub_rn(elevated[i], down)) ? (int)up : (int)down;
        sum += s.rem0[i];
        s.rank[i] = 0;
    }
    sum /= (D + 1);
#pragma unroll
    for (int i = 0; i < D; i++) {
        float di = __fsub_rn(elevated[i], (float)s.rem0[i]);
#pragma unroll
        for (int j = i + 1; j <= D; j++) {
            if (di < __fsub_rn(elevated[j], (float)s.rem0[j])) s.rank[i]++; else s.rank[j]++;
        }
    }
#pragma unroll
    for (int i = 0; i <= D; i++) {
        s.rank[i] += sum;
        if (s.rank[i] < 0) { s.rank[i] += D + 1; s.rem0[i] += D + 1; }
        else if (s.rank[i] > D) { s.rank[i] -= D + 1; s.rem0[i] -= D + 1; }
    }
#pragma unroll
    for (int i = 0; i <= D + 1; i++) s.bary[i] = 0.0f;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float delta = __fmul_rn(__fsub_rn(elevated[i], (float)s.rem0[i]), inv);
        // bary[D - rank] += delta ; bary[D + 1 - rank] -= delta   (static indexing to stay in registers)
#pragma unroll
        for (int r = 0; r <= D + 1; r++) {
            if (r == D - s.rank[i]) s.bary[r] = __fadd_rn(s.bary[r], delta);
            if (r == D + 1 - s.rank[i]) s.bary[r] = __fsub_rn(s.bary[r], delta);
        }
    }
    s.bary[0] = __fadd_rn(s.bary[0], __fadd_rn(1.0f, s.bary[D + 1]));
}

// d(bary)/d(direction): same scatter as the weights, applied to the elevated direction (weights are
// piecewise linear in x, so this is exact inside a simplex)
template <int D>
__device__ __forceinline__ void bary_tangent(const float* d_elev, const Simplex<D>& s, float* db) {
    const float inv = 1.0f / (float)(D + 1);
#pragma unroll
    for (int i = 0; i <= D + 1; i++) db[i] = 0.0f;
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float delta = d_elev[i] * inv;
#pragma unroll
        for (int r = 0; r <= D + 1; r++) {
            if (r == D - s.rank[i]) db[r] += delta;
            if (r == D + 1 - s.rank[i]) db[r] -= delta;
        }
    }
    db[0] += db[D + 1];
}

template <int D>
__device__ __forceinline__ unsigned vertex_index(const Simplex<D>& s, int r, const EncParams& p) {
    unsigned h = 0;
#pragma unroll
    for (int i = 0; i < D; i++) {
        int key = s.rem0[i] + r;
        if (s.rank[i] > D - r) key -= (D + 1);
        h += (unsigned)key;
        h *= 2531011u;
    }
    // h mod T without a division: umulhi(h, floor(2^32 / T)) is the quotient or one less -> one conditional subtraction
    const unsigned rem = h - __umulhi(h, p.cap_mask) * (unsigned)p.T;
    return rem >= (unsigned)p.T ? rem - (unsigned)p.T : rem;
}

// reverse of locate()'s weight scatter + elevation: dL/dbary[0..D] -> dL/dx (before the per-dim scale)
template <int D>
__device__ __forceinline__ void bary_grad_to_cf(float* dB /* size D+2, dB[D+1] must be 0 on entry */, const Simplex<D>& s,
                                                float* dcf) {
    const float inv = 1.0f / (float)(D + 1);
    dB[D + 1] += dB[0];
    float de[D + 1];
#pragma unroll
    for (int i = 0; i <= D; i++) {
        float a = 0.0f, b = 0.0f;
#pragma unroll
        for (int r = 0; r <= D + 1; r++) {
            if (r == D - s.rank[i]) a = dB[r];
            if (r == D + 1 - s.rank[i]) b = dB[r];
        }
        de[i] = (a - b) * inv;
    }
    // elevated[0] = sum_k cf[k]; elevated[i] = sum_{k>=i} cf[k] - i*cf[i-1]
    float run = 0.0f;
#pragma unroll
    for (int k = 0; k < D; k++) {
        run += de[k];
        dcf[k] = run - (float)(k + 1) * de[k + 1];
    }
}

// segmented sum over lanes that share a key (peers mask from __match_any_sync); result valid in the first peer
__device__ __forceinline__ float2 add_peers(unsigned peers, float2 x, int lane) {
    int rel = __popc(peers << (31 - lane) << 1);  // peers below me
    peers &= (0xfffffffeu << lane);
    while (__any_sync(kFull, peers)) {
        int next = __ffs(peers);
        float tx = __shfl_sync(kFull, x.x, (next - 1) & 31);
        float ty = __shfl_sync(kFull, x.y, (next - 1) & 31);
        if (next) { x.x += tx; x.y += ty; }
        int done = rel & 1;
        peers &= __ballot_sync(kFull, !done);
        rel >>= 1;
    }
    return x;
}
__device__ __forceinline__ void red_add_v2(float* addr, float2 v) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(v.x), "f"(v.y) : "memory");
}

struct LevelConsts {
    float scale[kMaxLevels * 4];
    float shift[kMaxLevels * 4];
    float window[kMaxLevels];
};
template <int D>
__device__ __forceinline__ void load_level_consts(LevelConsts& lc, const float* __restrict__ scale,
                                                  const float* __restrict__ shift, const float* __restrict__ window, int L) {
    for (int i = threadIdx.x; i < L * D; i += blockDim.x) {
        lc.scale[(i / D) * 4 + (i % D)] = scale[i];
        lc.shift[(i / D) * 4 + (i % D)] = shift ? shift[i] : 0.0f;
    }
    for (int i = threadIdx.x; i < L; i += blockDim.x) lc.window[i] = window ? window[i] : 1.0f;
}

// ------------------------------------------------------------------------------------------------ forward
template <int D>
__global__ void __launch_bounds__(kEncThreads)
k_enc_forward(EncParams p, const float* __restrict__ pos, const float2* __restrict__ lattice, const float* __restrict__ scale,
              const float* __restrict__ shift, const float* __restrict__ window, float* __restrict__ out) {
    // block = 32 consecutive samples x 4 level groups: warp g handles levels g, g+4, ... of the same 32 samples
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts lc;
    load_level_consts<D>(lc, scale, shift, window, p.L);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;                      // +1 float: conflict-free column writes
    float* tile = smem_dyn;
    const int n = blockIdx.x * 32 + lane;
    const bool valid = n < p.N;
    float x[D];
#pragma unroll
    for (int i = 0; i < D; i++) x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;

#pragma unroll 4
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], elevated[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * 4 + i]), lc.scale[l * 4 + i]);
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        const float2* tab = lattice + (size_t)l * p.T;
        float2 v[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) v[r] = __ldg(tab + vertex_index<D>(s, r, p));
        float w = lc.window[l];
        float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
        for (int r = 0; r <= D; r++) {
            float wr = s.bary[r] * w;
            a0 = fmaf(v[r].x, wr, a0);
            a1 = fmaf(v[r].y, wr, a1);
        }
        tile[lane * stride + 2 * l] = a0;
        tile[lane * stride + 2 * l + 1] = a1;
    }
    if (p.concat && warp == kGroups - 1) {
        const int base = 2 * p.L;
        for (int c = base; c < p.C; c++) {
            int d = c - base;
            float val = 0.0f;
#pragma unroll
            for (int i = 0; i < D; i++) if (i == d) val = x[i] * p.points_scaling;
            tile[lane * stride + c] = val;
        }
    }
    __syncthreads();
    // contiguous [rows, C] block of this CTA, written by all 128 threads
    const int row0 = blockIdx.x * 32;
    const int rows = min(32, p.N - row0);
    float* dst = out + (size_t)row0 * p.C;
    const int total = rows * p.C;
    for (int e = threadIdx.x; e < total; e += kEncThreads) {
        int r = e / p.C, c = e - r * p.C;
        dst[e] = tile[r * stride + c];
    }
}

// ------------------------------------------------------------------------------------------------ backward
// grad_lattice[l][idx][:] += window_l * bary_r * g[n][l][:]         (warp aggregated red.v2)
// grad_pos[n][j]          = sum_l window_l * sum_r (val_r . g_l) dB_r/dx_j  (+ concat columns)
template <int D, bool LATTICE, bool POS>
__global__ void __launch_bounds__(kEncThreads)
k_enc_backward(EncParams p, const float* __restrict__ pos, const float2* __restrict__ lattice, const float* __restrict__ scale,
               const float* __restrict__ shift, const float* __restrict__ window, const float* __restrict__ grad_out,
               float* __restrict__ grad_lattice, float* __restrict__ grad_pos) {
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts lc;
    __shared__ float red[kGroups][32][4];
    load_level_consts<D>(lc, scale, shift, window, p.L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;
    float* gtile = smem_dyn;                         // staged [32, C] block of grad_out (coalesced read)
    const int row0 = blockIdx.x * 32;
    {
        const int rows = min(32, p.N - row0);
        const float* src = grad_out + (size_t)row0 * p.C;
        for (int e = threadIdx.x; e < 32 * p.C; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            gtile[r * stride + c] = (r < rows) ? src[e] : 0.0f;
        }
    }
    __syncthreads();
    const int n = row0 + lane;
    const bool valid = n < p.N;
    float x[D], gp[D];
#pragma unroll
    for (int i = 0; i < D; i++) { x[i] = valid ? pos[(size_t)n * D + i] : 0.0f; gp[i] = 0.0f; }
    const float* g_row = gtile + lane * stride;

#pragma unroll 2
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], elevated[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * 4 + i]), lc.scale[l * 4 + i]);
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        float2 g = make_float2(g_row[2 * l], g_row[2 * l + 1]);
        float w = lc.window[l];
        unsigned idx[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) idx[r] = vertex_index<D>(s, r, p);
        if (POS) {
            const float2* tab = lattice + (size_t)l * p.T;
            float dB[D + 2];
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float2 v = __ldg(tab + idx[r]);
                dB[r] = w * (v.x * g.x + v.y * g.y);
            }
            dB[D + 1] = 0.0f;
            float dcf[D];
            bary_grad_to_cf<D>(dB, s, dcf);
#pragma unroll
            for (int i = 0; i < D; i++) gp[i] = fmaf(dcf[i], lc.scale[l * 4 + i], gp[i]);
        }
        if (LATTICE) {
            float* gtab = grad_lattice + (size_t)l * p.T * 2;
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float wr = s.bary[r] * w;
                float2 c = make_float2(g.x * wr, g.y * wr);
                unsigned key = valid ? idx[r] : 0xffffffffu;
                unsigned peers = __match_any_sync(kFull, key);
                c = add_peers(peers, c, lane);
                if (valid && lane == __ffs(peers) - 1) red_add_v2(gtab + (size_t)idx[r] * 2, c);
            }
        }
    }
    if (POS) {
        // sum the per-level-group partial position gradients of the 4 warps
#pragma unroll
        for (int i = 0; i < D; i++) red[warp][lane][i] = gp[i];
        __syncthreads();
        if (warp == 0 && valid) {
#pragma unroll
            for (int i = 0; i < D; i++) {
                float acc = red[0][lane][i];
#pragma unroll
                for (int w2 = 1; w2 < kGroups; w2++) acc += red[w2][lane][i];
                if (p.concat && 2 * p.L + i < p.C) acc = fmaf(g_row[2 * p.L + i], p.points_scaling, acc);
                grad_pos[(size_t)n * D + i] = acc;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ double backward
// Upstream gradient gg[n][j] flows into grad_pos. With dB_r = sum_j gg_j dB_r/dx_j (tangent of the weights):
//   grad_lattice[l][idx_r][:] += window_l * dB_r * g[n][l][:]
//   grad_grad_out[n][l][:]     = window_l * sum_r dB_r * val_r[:]      (concat columns: gg_j * scaling)
template <int D, bool LATTICE, bool GOUT>
__global__ void __launch_bounds__(kEncThreads)
k_enc_double_backward(EncParams p, const float* __restrict__ pos, const float2* __restrict__ lattice,
                      const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ window,
                      const float* __restrict__ gg_pos, const float* __restrict__ grad_out, float* __restrict__ grad_lattice,
                      float* __restrict__ grad_grad_out) {
    extern __shared__ float smem_dyn[];
    __shared__ LevelConsts lc;
    load_level_consts<D>(lc, scale, shift, window, p.L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int stride = p.C + 1;
    float* gtile = smem_dyn;                         // staged grad_out block
    float* otile = smem_dyn + 32 * stride;           // grad_grad_out block, written out coalesced
    const int row0 = blockIdx.x * 32;
    const int rows = min(32, p.N - row0);
    if (LATTICE) {
        const float* src = grad_out + (size_t)row0 * p.C;
        for (int e = threadIdx.x; e < 32 * p.C; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            gtile[r * stride + c] = (r < rows) ? src[e] : 0.0f;
        }
    }
    __syncthreads();
    const int n = row0 + lane;
    const bool valid = n < p.N;
    float x[D], u[D];
#pragma unroll
    for (int i = 0; i < D; i++) {
        x[i] = valid ? pos[(size_t)n * D + i] : 0.0f;
        u[i] = valid ? gg_pos[(size_t)n * D + i] : 0.0f;
    }
#pragma unroll 2
    for (int l = warp; l < p.L; l += kGroups) {
        float cf[D], dcf[D], elevated[D + 1], d_elev[D + 1];
#pragma unroll
        for (int i = 0; i < D; i++) {
            cf[i] = __fmul_rn(__fadd_rn(x[i], lc.shift[l * 4 + i]), lc.scale[l * 4 + i]);
            dcf[i] = u[i] * lc.scale[l * 4 + i];
        }
        elevate<D>(cf, elevated);
        Simplex<D> s;
        locate<D>(elevated, s);
        {
            float sm = 0.0f;
#pragma unroll
            for (int i = D; i > 0; i--) { d_elev[i] = sm - (float)i * dcf[i - 1]; sm += dcf[i - 1]; }
            d_elev[0] = sm;
        }
        float db[D + 2];
        bary_tangent<D>(d_elev, s, db);
        float w = lc.window[l];
        unsigned idx[D + 1];
#pragma unroll
        for (int r = 0; r <= D; r++) idx[r] = vertex_index<D>(s, r, p);
        if (GOUT) {
            const float2* tab = lattice + (size_t)l * p.T;
            float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float2 v = __ldg(tab + idx[r]);
                float c = db[r] * w;
                a0 = fmaf(v.x, c, a0);
                a1 = fmaf(v.y, c, a1);
            }
            otile[lane * stride + 2 * l] = a0;
            otile[lane * stride + 2 * l + 1] = a1;
        }
        if (LATTICE) {
            float2 g = make_float2(gtile[lane * stride + 2 * l], gtile[lane * stride + 2 * l + 1]);
            float* gtab = grad_lattice + (size_t)l * p.T * 2;
#pragma unroll
            for (int r = 0; r <= D; r++) {
                float c = db[r] * w;
                float2 cv = make_float2(g.x * c, g.y * c);
                unsigned key = valid ? idx[r] : 0xffffffffu;
                unsigned peers = __match_any_sync(kFull, key);
                cv = add_peers(peers, cv, lane);
                if (valid && lane == __ffs(peers) - 1) red_add_v2(gtab + (size_t)idx[r] * 2, cv);
            }
        }
    }
    if (GOUT) {
        if (p.concat && warp == kGroups - 1) {
            const int base = 2 * p.L;
            for (int c = base; c < p.C; c++) {
                int d = c - base;
                float val = 0.0f;
#pragma unroll
                for (int i = 0; i < D; i++) if (i == d) val = u[i] * p.points_scaling;
                otile[lane * stride + c] = val;
            }
        }
        __syncthreads();
        float* dst = grad_grad_out + (size_t)row0 * p.C;
        const int total = rows * p.C;
        for (int e = threadIdx.x; e < total; e += kEncThreads) {
            int r = e / p.C, c = e - r * p.C;
            dst[e] = otile[r * stride + c];
        }
    }
}

inline int make_params(EncParams& p, int N, int D, int L, int F, int T, int concat, float points_scaling) {
    if (F != 2 || (D != 3 && D != 4) || L < 1 || L > kMaxLevels || T < 1) return PSDF_ERR_UNSUPPORTED;
    p.N = N; p.L = L; p.T = T;
    int E = concat ? (D + F - 1) / F : 0;
    p.C = (L + E) * F;
    p.concat = concat;
    p.points_scaling = points_scaling;
    p.cap_mask = T <= 1 ? 0xffffffffu : (unsigned)(0x100000000ull / (unsigned long long)(unsigned)T);
    return PSDF_OK;
}
#define ST ((cudaStream_t)stream)
}  // namespace

extern "C" {

int psdf_enc_forward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                     const float* shift, const float* window, int concat_points, float points_scaling, float* out, void* stream) {
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (N == 0) return PSDF_OK;
    int blocks = div_up(N, 32);
    size_t smem = (size_t)32 * (p.C + 1) * sizeof(float);
    const float2* lat = reinterpret_cast<const float2*>(lattice);
    if (D == 3) k_enc_forward<3><<<blocks, kEncThreads, smem, ST>>>(p, pos, lat, scale_factor, shift, window, out);
    else k_enc_forward<4><<<blocks, kEncThreads, smem, ST>>>(p, pos, lat, scale_factor, shift, window, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_enc_backward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                      const float* shift, const float* window, int concat_points, float points_scaling, const float* grad_out,
                      float* grad_lattice, float* grad_pos, void* stream) {
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (N == 0 || (!grad_lattice && !grad_pos)) return PSDF_OK;
    int blocks = div_up(N, 32);
    size_t smem = (size_t)32 * (p.C + 1) * sizeof(float);
    const float2* lat = reinterpret_cast<const float2*>(lattice);
#define LAUNCH_BWD(DD, LA, PO) \
    k_enc_backward<DD, LA, PO><<<blocks, kEncThreads, smem, ST>>>(p, pos, lat, scale_factor, shift, window, grad_out, grad_lattice, grad_pos)
    if (D == 3) {
        if (grad_lattice && grad_pos) LAUNCH_BWD(3, true, true);
        else if (grad_lattice) LAUNCH_BWD(3, true, false);
        else LAUNCH_BWD(3, false, true);
    } else {
        if (grad_lattice && grad_pos) LAUNCH_BWD(4, true, true);
        else if (grad_lattice) LAUNCH_BWD(4, true, false);
        else LAUNCH_BWD(4, false, true);
    }
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_enc_double_backward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                             const float* shift, const float* window, int concat_points, float points_scaling,
                             const float* gg_pos, const float* grad_out, float* grad_lattice, float* grad_grad_out, void* stream) {
    EncParams p;
    int rc = make_params(p, N, D, L, F, T, concat_points, points_scaling);
    if (rc) return rc;
    if (N == 0 || (!grad_lattice && !grad_grad_out)) return PSDF_OK;
    int blocks = div_up(N, 32);
    size_t smem = (size_t)2 * 32 * (p.C + 1) * sizeof(float);
    const float2* lat = reinterpret_cast<const float2*>(lattice);
#define LAUNCH_DBL(DD, LA, GO)                                                                                                  \
    k_enc_double_backward<DD, LA, GO><<<blocks, kEncThreads, smem, ST>>>(p, pos, lat, scale_factor, shift, window, gg_pos, grad_out, \
                                                                     grad_lattice, grad_grad_out)
    if (D == 3) {
        if (grad_lattice && grad_grad_out) LAUNCH_DBL(3, true, true);
        else if (grad_lattice) LAUNCH_DBL(3, true, false);
        else LAUNCH_DBL(3, false, true);
    } else {
        if (grad_lattice && grad_grad_out) LAUNCH_DBL(4, true, true);
        else if (grad_lattice) LAUNCH_DBL(4, true, false);
        else LAUNCH_DBL(4, false, true);
    }
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_abi_version(void) { return PSDF_ABI_VERSION; }
int psdf_device_ok(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); return 0; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, 0) != cudaSuccess) return 0;
    return prop.major == 9 ? 1 : 0;
}

}  // extern "C"
