// Ray-path kernels for sm_90a: bounding sphere, occupancy grid (Morton DDA), packed sample
// containers, fg/bg ray samplers, spherical harmonics and ray generation.
// Compiled with -fmad=false: every FMA below is explicit and placed where the reference's nvcc build
// contracts (see common.cuh). Reference semantics cited per kernel.
//
// Work mapping: the voxel walk is a serial float recurrence (t += step + eps) that must be reproduced
// bit-for-bit, but the occupancy bytes do not feed it. The sampler used in training runs one WARP per ray with
// speculative 32-step windows (see k_occ_samples_in_occupied); the first-sample / advance marchers of sphere tracing
// are one thread per ray with an 8-step look-ahead of the recurrence over the loads (common.cuh). Copy/packing
// kernels are warp-per-ray with coalesced accesses. Slots in the sample pool are deterministic (ray * stride) rather than handed out
// by a global atomic (SURVEY.md F8), with the reference's atomic order available as slot_mode=0.
#include "common.cuh"
#include "sh.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxSteps = 4096;  // OccupancyGridGPU.cuh:24

// ------------------------------------------------------------------------------------------------ Sphere
// SphereGPU.cuh:21-93. FMA placement copied from the reference SASS: dot(a,b)=fma(az,bz,fma(ax,bx,ay*by)).
__global__ void __launch_bounds__(kThreads) k_sphere_ray_intersection(int n, float radius, float cx, float cy, float cz,
                                                                      const float* __restrict__ origins,
                                                                      const float* __restrict__ dirs, float* __restrict__ pe,
                                                                      float* __restrict__ te, float* __restrict__ px,
                                                                      float* __restrict__ tx, uint8_t* __restrict__ hit) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float ox = origins[3 * i], oy = origins[3 * i + 1], oz = origins[3 * i + 2];
    float dx = dirs[3 * i], dy = dirs[3 * i + 1], dz = dirs[3 * i + 2];
    float qx = __fsub_rn(ox, cx), qy = __fsub_rn(oy, cy), qz = __fsub_rn(oz, cz);
    float a = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    float bh = __fmaf_rn(dz, qz, __fmaf_rn(dx, qx, __fmul_rn(dy, qy)));
    float b = __fadd_rn(bh, bh);
    float c = __fmaf_rn(-radius, radius, __fmaf_rn(qz, qz, __fmaf_rn(qx, qx, __fmul_rn(qy, qy))));
    float disc = __fmaf_rn(b, b, __fmul_rn(__fmul_rn(a, -4.0f), c));
    float sq = __fsqrt_rn(fabsf(disc));
    double den = 2.0 * (double)a;
    float t0 = (float)((double)__fsub_rn(-b, sq) / den);
    float t1 = (float)((double)__fadd_rn(-b, sq) / den);
    bool miss = disc < 0.0f;
    if (miss) { t0 = 0.0f; t1 = 0.0f; }
    t0 = fmaxf(0.0f, t0);
    pe[3 * i] = __fmaf_rn(dx, t0, ox); pe[3 * i + 1] = __fmaf_rn(dy, t0, oy); pe[3 * i + 2] = __fmaf_rn(dz, t0, oz);
    px[3 * i] = __fmaf_rn(dx, t1, ox); px[3 * i + 1] = __fmaf_rn(dy, t1, oy); px[3 * i + 2] = __fmaf_rn(dz, t1, oz);
    te[i] = t0;
    tx[i] = t1;
    hit[i] = miss ? 0 : 1;
}
// SphereGPU.cuh:96-130 (the centre is not added, like the reference)
__global__ void __launch_bounds__(kThreads) k_sphere_rand_points(int n, float radius, const float* __restrict__ phi,
                                                                 const float* __restrict__ ct, const float* __restrict__ u,
                                                                 float* __restrict__ pts) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float theta = acosf(ct[i]);
    float r = radius * (float)pow((double)u[i], 1.0 / 3);
    float st = sinf(theta);
    pts[3 * i] = r * st * cosf(phi[i]);
    pts[3 * i + 1] = r * st * sinf(phi[i]);
    pts[3 * i + 2] = r * cosf(theta);
}
// Sphere.cu:111-119 : ||p - c|| < radius
__global__ void __launch_bounds__(kThreads) k_sphere_inside(int n, float radius, float cx, float cy, float cz,
                                                            const float* __restrict__ p, uint8_t* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = p[3 * i] - cx, y = p[3 * i + 1] - cy, z = p[3 * i + 2] - cz;
    out[i] = sqrtf(x * x + y * y + z * z) < radius;
}

// advance a device-resident pcg32 {state, inc} (the host-side `rng.advance(2^32)` after every jittered call)
__global__ void k_rng_advance(uint64_t* rng_dev, long long delta) {
    Pcg32 r(rng_dev[0], rng_dev[1]);
    r.advance(delta);
    rng_dev[0] = r.state;
}
// ------------------------------------------------------------------------------------------------ Occupancy
// OccupancyGridGPU.cuh:196-301
__global__ void __launch_bounds__(kThreads) k_occ_grid_points(int n, GridGeom g, const int* __restrict__ idx, Pcg32 rng,
                                                              bool randomize, float* __restrict__ out) {
    rng.resolve();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t v = idx ? (uint32_t)idx[i] : (uint32_t)i;
    float3 p = voxel_to_pos(v, g, true);
    if (randomize) {
        float vs = __fdiv_rn(g.extent, (float)g.V);
        float half = __fmul_rn(vs, 0.5f);
        rng.advance((int64_t)(i * 3));
        p.x = __fadd_rn(p.x, __fmaf_rn(rng.next_float(), vs, -half));
        p.y = __fadd_rn(p.y, __fmaf_rn(rng.next_float(), vs, -half));
        p.z = __fadd_rn(p.z, __fmaf_rn(rng.next_float(), vs, -half));
    }
    out[3 * i] = p.x; out[3 * i + 1] = p.y; out[3 * i + 2] = p.z;
}
// A random update sample may hold a voxel more than once, and then whichever thread stores last wins, as in the reference. In
// deterministic mode (common.cuh) the LAST sample of a voxel in sample order wins instead, what a sequential loop over the sample
// does: k_occ_claim records 1 + the highest sample index per voxel in `winner`, and only that sample writes (and clears the record).
__global__ void __launch_bounds__(kThreads) k_occ_claim(int n, const int* __restrict__ idx, int* __restrict__ winner, long long voxels) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && idx[i] < voxels) atomicMax(&winner[idx[i]], i + 1);
}
__device__ __forceinline__ bool occ_wins(int* winner, long long voxels, int i, int v) {
    if (!winner || v >= voxels) return true;       // no arbitration (default, or a voxel beyond the reserved grid)
    if (winner[v] != i + 1) return false;
    winner[v] = 0;
    return true;
}
// OccupancyGridGPU.cuh:303-378
__global__ void __launch_bounds__(kThreads) k_occ_update_density(int n, const float* __restrict__ density,
                                                                 const int* __restrict__ idx, float decay, float thresh,
                                                                 float* __restrict__ values, uint8_t* __restrict__ occ, int* __restrict__ winner,
                                                             long long voxels) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int v = idx ? idx[i] : i;
    if (!occ_wins(winner, voxels, i, v)) return;
    float upd = fmaxf(density[i], __fmul_rn(values[v], decay));
    values[v] = upd;
    occ[v] = upd > thresh;
}
// OccupancyGridGPU.cuh:381-507 ; logistic pdf s*e/(1+e)^2 with e=exp(-s*x)
__global__ void __launch_bounds__(kThreads) k_occ_update_sdf(int n, const float* __restrict__ sdf, const int* __restrict__ idx,
                                                             float range, float inv_s_scalar,
                                                             const float* __restrict__ inv_s_dev, float thresh,
                                                             float* __restrict__ values, uint8_t* __restrict__ occ, int* __restrict__ winner,
                                                             long long voxels) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int v = idx ? idx[i] : i;
    if (!occ_wins(winner, voxels, i, v)) return;
    float s = sdf[i];
    values[v] = s;
    float inv_s = inv_s_dev ? inv_s_dev[0] : inv_s_scalar;
    float capped = clampf(fabsf(s) - range, 0.0f, 1e10f);
    float e = expf(-inv_s * capped);
    float w = inv_s * e / powf(1.0f + e, 2.0f);
    occ[v] = w > thresh;
}
// OccupancyGridGPU.cuh:901-941
__global__ void __launch_bounds__(kThreads) k_occ_check(int n, GridGeom g, const uint8_t* __restrict__ occ,
                                                        const float* __restrict__ pts, uint8_t* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int nv = g.V * g.V * g.V;
    int v = pos_to_voxel(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], g);
    bool oob = v > (nv - 1) || v < 0;
    out[i] = oob ? 0 : occ[v];
}

struct RayIn {
    float ox, oy, oz, dx, dy, dz, ix, iy, iz;
};
__device__ __forceinline__ RayIn load_ray(const float* __restrict__ origins, const float* __restrict__ dirs, int i) {
    RayIn r;
    r.ox = origins[3 * i]; r.oy = origins[3 * i + 1]; r.oz = origins[3 * i + 2];
    r.dx = dirs[3 * i]; r.dy = dirs[3 * i + 1]; r.dz = dirs[3 * i + 2];
    r.ix = safe_inv(r.dx); r.iy = safe_inv(r.dy); r.iz = safe_inv(r.dz);
    return r;
}

// OccupancyGridGPU.cuh:510-703
// slot_mode 1: ray i owns slots [i*max_per_ray, (i+1)*max_per_ray) (deterministic); 0: global atomic like the reference.
//
// One WARP per ray. The reference runs two serial marches per ray (one thread each); here the scalar recurrences are kept
// bit for bit, but every lane replays them ("uniform serial") so that the memory work hangs off them 32 wide:
//   pass 1 (length inside occupied voxels): the DDA chain t <- t + dn(t) + eps advances 32 steps per window, lane k latches
//     step k's voxel and fetches its occupancy, so a window costs ONE load latency; the length is then accumulated in the
//     original order over the occupied steps;
//   pass 2 (sample creation): a window speculates that the next w iterations all emit a sample (t advances by `spacing`),
//     lane j evaluates iteration j (position, voxel, occupancy load, sample stores) and a ballot finds the first iteration
//     that does not emit; that iteration (skip to the next voxel, with its jitter draw) is then executed serially.
// The march stops once all n_create samples exist: the reference keeps stepping to t_exit, which changes no output.
constexpr int kOccWarpsPerBlock = 4;
template <bool kInvMul>
__global__ void __launch_bounds__(kOccWarpsPerBlock * 32)
k_occ_samples_in_occupied(int nr_rays, GridGeom g, const float* __restrict__ origins, const float* __restrict__ dirs,
                          const float* __restrict__ t_entry, const float* __restrict__ t_exit_,
                          const uint8_t* __restrict__ occ, float min_dist, int max_per_ray, int max_nr_samples, Pcg32 rng,
                          bool jitter, int slot_mode, float* __restrict__ s_pos, float* __restrict__ s_dirs,
                          float* __restrict__ s_z, float* __restrict__ s_dt, float* __restrict__ ray_fixed_dt,
                          int* __restrict__ start_end, int* __restrict__ cur_nr_samples) {
    rng.resolve();
    const unsigned kFull = 0xffffffffu;
    const int idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (idx >= nr_rays) return;
    const int nv = g.V * g.V * g.V;
    const float eps = 1e-6f;
    RayIn r = load_ray(origins, dirs, idx);
    const float t_start = t_entry[idx], t_exit = t_exit_[idx];
    const float hsx = half_sign(r.dx), hsy = half_sign(r.dy), hsz = half_sign(r.dz);
    const float Vf = (float)g.V, inv_V = 1.0f / Vf;       // V is a power of two: t / V == t * (1 / V) exactly

    // ---- pass 1. A window runs 32 DDA steps with no control dependence on the voxel index (steps past the end of the
    // march are computed and discarded), lane k latches step k; the occupancy bytes of window i are consumed after the chain
    // of window i+1, so their latency hides behind it.
    float t = t_start;
    int steps = 0;
    float occ_len = 0.0f;
    bool alive = (t < t_exit);
    unsigned p_o = 0;                 // previous window: occupancy byte of this lane's step (0 if the step was not recorded)
    float p_dn = 0.f, p_t = 0.f;
    auto consume = [&](unsigned o, float dn, float tt) {
        unsigned hits = __ballot_sync(kFull, o != 0);
        while (hits) {                                   // occupied steps, in march order
            const int k = __ffs(hits) - 1;
            hits &= hits - 1;
            const float dnk = __shfl_sync(kFull, dn, k), tk = __shfl_sync(kFull, tt, k);
            occ_len = __fadd_rn(occ_len, dnk);
            const float tm = __fsub_rn(tk, eps);
            if (tm > t_exit) occ_len = __fsub_rn(occ_len, __fsub_rn(tm, t_exit));
        }
    };
    while (alive) {
        // the chain carries only what the recurrence needs (position -> DDA step -> t); lane k latches the t at the start of
        // step k and its step length, and derives its voxel (Morton index) from that t afterwards, 32 lanes in parallel
        float myt0 = 0.f, mydn = 0.f;
        float tw = t;
#pragma unroll 8
        for (int k = 0; k < 32; k++) {
            const float px = __fmaf_rn(r.dx, tw, r.ox), py = __fmaf_rn(r.dy, tw, r.oy), pz = __fmaf_rn(r.dz, tw, r.oz);
            const float dn = dda_step_s(px, py, pz, hsx, hsy, hsz, r.ix, r.iy, r.iz, Vf, inv_V);
            if (lane == k) { myt0 = tw; mydn = dn; }
            tw = __fadd_rn(__fadd_rn(tw, dn), eps);
        }
        float myt = __shfl_down_sync(kFull, myt0, 1);           // t after this lane's step = t at the start of the next one
        if (lane == 31) myt = tw;
        const int myv = pos_to_voxel_t<kInvMul>(__fmaf_rn(r.dx, myt0, r.ox), __fmaf_rn(r.dy, myt0, r.oy), __fmaf_rn(r.dz, myt0, r.oz), g, Vf);
        const bool myoob = (myv >= nv || myv < 0);
        // step k+1 is attempted iff step k was inside the grid and left the march alive
        const bool last = myoob || !(myt < t_exit) || !(steps + lane + 1 < kMaxSteps);
        const unsigned stop = __ballot_sync(kFull, last);
        const int first = stop ? __ffs(stop) - 1 : 32;
        int m = 32;
        if (first < 32) { m = __shfl_sync(kFull, (int)myoob, first) ? first : first + 1; alive = false; }
        if (m > 0) t = __shfl_sync(kFull, myt, m - 1);
        steps += m;
        const unsigned o = (lane < m) ? (unsigned)__ldg(occ + myv) : 0u;     // consumed one window later
        consume(p_o, p_dn, p_t);
        p_o = o; p_dn = mydn; p_t = myt;
    }
    consume(p_o, p_dn, p_t);

    int n_create = (int)__fdiv_rn(occ_len, min_dist);
    n_create = min(max(n_create, 0), max_per_ray);
    const float spacing = __fdiv_rn(occ_len, (float)n_create);

    if (n_create > 1) {
        int start = 0;
        if (lane == 0) {
            if (slot_mode == 1) { start = idx * max_per_ray; atomicAdd(cur_nr_samples, n_create); }
            else start = atomicAdd(cur_nr_samples, n_create);
        }
        start = __shfl_sync(kFull, start, 0);
        if (start + n_create > max_nr_samples) {
            if (lane == 0) { start_end[2 * idx] = start; start_end[2 * idx + 1] = start + n_create; ray_fixed_dt[idx] = spacing; }
            return;
        }
        t = t_start;
        steps = 0;
        if (jitter) {
            rng.advance(idx);
            t = __fmaf_rn(rng.next_float(), spacing, t);
        }
        int created = 0;
        float last_z = 0.0f;
        while (t < t_exit && steps < kMaxSteps && created < n_create) {
            // ---- emit window: the next w iterations are assumed to create a sample each (t advances by the spacing)
            const int w = min(32, n_create - created);
            float tj = t, mine = t;
            for (int j = 1; j < w; j++) { tj = __fadd_rn(tj, spacing); if (lane == j) mine = tj; }
            const bool in = (lane < w) && (mine < t_exit) && (steps + lane < kMaxSteps);
            const float tc = clampf(mine, t_start, t_exit);
            const float px = __fmaf_rn(r.dx, tc, r.ox), py = __fmaf_rn(r.dy, tc, r.oy), pz = __fmaf_rn(r.dz, tc, r.oz);
            const int v = pos_to_voxel_t<kInvMul>(px, py, pz, g, Vf);
            const bool inside = in && !(v >= nv || v < 0);
            const bool emit = inside && __ldg(occ + v);
            const unsigned nem = ~__ballot_sync(kFull, emit);
            const int e = min(nem ? __ffs(nem) - 1 : 32, w);                 // leading iterations that emit
            if (lane < e) {
                const int s = start + created + lane;
                s_pos[3 * s] = px; s_pos[3 * s + 1] = py; s_pos[3 * s + 2] = pz;
                s_dirs[3 * s] = r.dx; s_dirs[3 * s + 1] = r.dy; s_dirs[3 * s + 2] = r.dz;
                s_z[s] = tc;
                s_dt[s] = spacing;
            }
            if (e > 0) {
                last_z = __shfl_sync(kFull, tc, e - 1);
                for (int j = 0; j < e; j++) t = __fadd_rn(clampf(t, t_start, t_exit), spacing);
                created += e;
                steps += e;
            }
            if (e == w) continue;
            // iteration e does not emit: it ends the march (t_exit / step limit / outside the grid) or starts a run of skips
            if (!__shfl_sync(kFull, (int)inside, e)) break;
            // ---- skip windows: the next 32 iterations are assumed to skip to the next voxel (DDA step + jitter draw); lane k
            // latches the state at the START of iteration k and tests that position; the first iteration that would not skip
            // (occupied voxel, end of the march) is where the state is rolled back to
            bool finished = false;
            while (true) {
                float myt = 0.f;
                uint64_t myrng = 0;
                float tw = t;
#pragma unroll 4
                for (int k = 0; k < 32; k++) {
                    if (lane == k) { myt = tw; myrng = rng.state; }
                    const float tk = clampf(tw, t_start, t_exit);
                    const float qx = __fmaf_rn(r.dx, tk, r.ox), qy = __fmaf_rn(r.dy, tk, r.oy), qz = __fmaf_rn(r.dz, tk, r.oz);
                    float delta = dda_step_s(qx, qy, qz, hsx, hsy, hsz, r.ix, r.iy, r.iz, Vf, inv_V);
                    if (jitter) delta = __fmaf_rn(rng.next_float(), spacing, delta);
                    tw = __fadd_rn(__fadd_rn(tk, delta), eps);
                }
                const float mtk = clampf(myt, t_start, t_exit);
                const int myv2 = pos_to_voxel_t<kInvMul>(__fmaf_rn(r.dx, mtk, r.ox), __fmaf_rn(r.dy, mtk, r.oy), __fmaf_rn(r.dz, mtk, r.oz), g, Vf);
                const bool myoob2 = (myv2 >= nv || myv2 < 0);
                const bool in2 = (myt < t_exit) && (steps + lane < kMaxSteps);
                const bool occ2 = in2 && !myoob2 && __ldg(occ + myv2);
                const unsigned stop2 = __ballot_sync(kFull, !in2 || myoob2 || occ2);
                const int f = stop2 ? __ffs(stop2) - 1 : 32;
                if (f == 32) {                       // 32 confirmed skips; the generator already sits after the 32nd draw
                    t = tw;
                    steps += 32;
                    if (!(t < t_exit && steps < kMaxSteps)) { finished = true; break; }
                    continue;
                }
                t = __shfl_sync(kFull, myt, f);
                const uint32_t lo = __shfl_sync(kFull, (uint32_t)myrng, f), hi = __shfl_sync(kFull, (uint32_t)(myrng >> 32), f);
                rng.state = ((uint64_t)hi << 32) | lo;
                steps += f;
                finished = !__shfl_sync(kFull, (int)occ2, f);      // stopped by the end of the march, not by an occupied voxel
                break;
            }
            if (finished) break;
        }
        for (int i = created + lane; i < n_create; i += 32) {
            const int s = start + i;
            s_pos[3 * s] = 0; s_pos[3 * s + 1] = 0; s_pos[3 * s + 2] = 0;
            s_dirs[3 * s] = 0; s_dirs[3 * s + 1] = 0; s_dirs[3 * s + 2] = 0;
            s_z[s] = -1.0f;
            s_dt[s] = 0;
        }
        __syncwarp();
        if (lane == 0) {
            if (created > 0) s_dt[start + created - 1] = clampf(__fsub_rn(t_exit, last_z), 0.0f, spacing);
            if (created <= 2) { ray_fixed_dt[idx] = 0; start_end[2 * idx] = 0; start_end[2 * idx + 1] = 0; }
            else { ray_fixed_dt[idx] = spacing; start_end[2 * idx] = start; start_end[2 * idx + 1] = start + created; }
        }
    } else if (lane == 0) {
        ray_fixed_dt[idx] = 0;
        start_end[2 * idx] = 0;
        start_end[2 * idx + 1] = 0;
    }
}

// OccupancyGridGPU.cuh:707-814 ; one sample at the first occupied voxel. slot_mode 1: slot == ray index.
__global__ void __launch_bounds__(kThreads)
k_occ_first_sample(int nr_rays, GridGeom g, const float* __restrict__ origins, const float* __restrict__ dirs,
                   const float* __restrict__ t_entry, const float* __restrict__ t_exit_, const uint8_t* __restrict__ occ,
                   int max_nr_samples, int slot_mode, float* __restrict__ s_pos, float* __restrict__ s_dirs,
                   float* __restrict__ s_z, float* __restrict__ s_dt, float* __restrict__ ray_fixed_dt,
                   int* __restrict__ start_end, int* __restrict__ cur_nr_samples) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nr_rays) return;
    const int nv = g.V * g.V * g.V;
    const float eps = 1e-6f;
    RayIn r = load_ray(origins, dirs, idx);
    float t = t_entry[idx], t_exit = t_exit_[idx];
    // the reference loop never increments nr_steps (:759-798); t grows by >= eps per step so it ends.
    while (t < t_exit) {
        float px = __fmaf_rn(r.dx, t, r.ox), py = __fmaf_rn(r.dy, t, r.oy), pz = __fmaf_rn(r.dz, t, r.oz);
        int v = pos_to_voxel(px, py, pz, g);
        if (v >= nv || v < 0) break;
        float dn = dda_step(px, py, pz, r.dx, r.dy, r.dz, r.ix, r.iy, r.iz, g.V);
        t = __fadd_rn(__fadd_rn(t, dn), eps);
        if (__ldg(occ + v)) {
            int start;
            if (slot_mode == 1) { start = idx; atomicAdd(cur_nr_samples, 1); }
            else start = atomicAdd(cur_nr_samples, 1);
            start_end[2 * idx] = start;
            start_end[2 * idx + 1] = start + 1;
            ray_fixed_dt[idx] = 0;
            if (start + 1 > max_nr_samples) return;
            s_pos[3 * start] = px; s_pos[3 * start + 1] = py; s_pos[3 * start + 2] = pz;
            s_dirs[3 * start] = r.dx; s_dirs[3 * start + 1] = r.dy; s_dirs[3 * start + 2] = r.dz;
            s_z[start] = t;  // already advanced t, as in the reference (:766,790)
            s_dt[start] = 0;
            return;
        }
    }
    ray_fixed_dt[idx] = 0;
    start_end[2 * idx] = 0;
    start_end[2 * idx + 1] = 0;
}

// OccupancyGridGPU.cuh:817-895 ; in-place update of pos (output aliases input, OccupancyGrid.cu:311)
__global__ void __launch_bounds__(kThreads)
k_occ_advance_to_next_occupied(int n, GridGeom g, const float* __restrict__ dirs, float* __restrict__ pos_io,
                               const uint8_t* __restrict__ occ, uint8_t* __restrict__ within) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    float px = pos_io[3 * idx], py = pos_io[3 * idx + 1], pz = pos_io[3 * idx + 2];
    // the march lives in common.cuh (shared with the fused sphere tracer); it leaves the position as it was when its step budget runs out
    const bool wb = occ_advance_to_next_occupied(g, occ, px, py, pz, dirs[3 * idx], dirs[3 * idx + 1], dirs[3 * idx + 2]);
    pos_io[3 * idx] = px; pos_io[3 * idx + 1] = py; pos_io[3 * idx + 2] = pz;
    within[idx] = wb ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ RaySampler
// RaySamplerGPU.cuh:162-335
__global__ void __launch_bounds__(kThreads)
k_sampler_fg(int nr_rays, const float* __restrict__ origins, const float* __restrict__ dirs, const float* __restrict__ t_entry,
             const float* __restrict__ t_exit_, float min_dist, int max_per_ray, int max_nr_samples, Pcg32 rng, bool jitter,
             int slot_mode, float* __restrict__ s_pos, float* __restrict__ s_dirs, float* __restrict__ s_z,
             float* __restrict__ s_dt, float* __restrict__ ray_fixed_dt, int* __restrict__ start_end,
             int* __restrict__ cur_nr_samples) {
    rng.resolve();
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nr_rays) return;
    const float eps = 1e-6f;
    float ox = origins[3 * idx], oy = origins[3 * idx + 1], oz = origins[3 * idx + 2];
    float dx = dirs[3 * idx], dy = dirs[3 * idx + 1], dz = dirs[3 * idx + 2];
    float t_start = t_entry[idx], t_exit = t_exit_[idx];
    float len = __fsub_rn(t_exit, t_start);
    int n_create = (int)__fdiv_rn(len, min_dist);
    n_create = min(max(n_create, 0), max_per_ray);
    float spacing = __fdiv_rn(len, (float)n_create);
    if (n_create > 1 && len > eps) {
        int start;
        if (slot_mode == 1) { start = idx * max_per_ray; atomicAdd(cur_nr_samples, n_create); }
        else start = atomicAdd(cur_nr_samples, n_create);
        start_end[2 * idx] = start;
        start_end[2 * idx + 1] = start + n_create;
        ray_fixed_dt[idx] = spacing;
        if (start + n_create > max_nr_samples) return;
        float t = t_start;
        int steps = 0;
        if (jitter) {
            rng.advance(idx);
            t = __fmaf_rn(rng.next_float(), spacing, t);
        }
        int created = 0;
        float last_z = 0;
        while (t < t_exit && steps < kMaxSteps) {
            t = clampf(t, t_start, t_exit);
            if (created < n_create) {
                int s = start + created;
                s_pos[3 * s] = __fmaf_rn(dx, t, ox); s_pos[3 * s + 1] = __fmaf_rn(dy, t, oy); s_pos[3 * s + 2] = __fmaf_rn(dz, t, oz);
                s_dirs[3 * s] = dx; s_dirs[3 * s + 1] = dy; s_dirs[3 * s + 2] = dz;
                s_z[s] = t;
                s_dt[s] = spacing;
                last_z = t;
                t = __fadd_rn(t, spacing);
                created++;
            }
            steps++;
        }
        if (created > 0) s_dt[start + created - 1] = clampf(__fsub_rn(t_exit, last_z), 0.0f, spacing);
        for (int i = created; i < n_create; i++) {
            int s = start + i;
            s_pos[3 * s] = 0; s_pos[3 * s + 1] = 0; s_pos[3 * s + 2] = 0;
            s_dirs[3 * s] = 0; s_dirs[3 * s + 1] = 0; s_dirs[3 * s + 2] = 0;
            s_z[s] = -1.0f;
            s_dt[s] = 0;
        }
        start_end[2 * idx + 1] = start + created;
        if (created <= 2) {
            ray_fixed_dt[idx] = 0;
            start_end[2 * idx] = 0;
            start_end[2 * idx + 1] = 0;
        }
    } else {
        ray_fixed_dt[idx] = 0;
        start_end[2 * idx] = 0;
        start_end[2 * idx + 1] = 0;
    }
}

// RaySamplerGPU.cuh:37-158 ; inverse-depth background samples with the NeRF++ 4-D parametrisation.
// The per-sample cumulative rng.advance(idx*n) of the reference (:88-94) is kept.
__global__ void __launch_bounds__(kThreads)
k_sampler_bg(int nr_rays, int n_per_ray, const float* __restrict__ origins, const float* __restrict__ dirs,
             const float* __restrict__ t_exit_, float sphere_radius, float cx, float cy, float cz, Pcg32 rng, bool randomize,
             bool contract, float* __restrict__ s3, float* __restrict__ s4, float* __restrict__ s_dirs,
             float* __restrict__ s_z, float* __restrict__ s_dt, float* __restrict__ ray_fixed_dt,
             int* __restrict__ start_end) {
    rng.resolve();
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nr_rays) return;
    float ox = origins[3 * idx], oy = origins[3 * idx + 1], oz = origins[3 * idx + 2];
    float dx = dirs[3 * idx], dy = dirs[3 * idx + 1], dz = dirs[3 * idx + 2];
    float t_exit = t_exit_[idx];
    const float min_t = 1e-3f;
    float t_between = (float)((1.0 - (double)min_t) / (double)(n_per_ray - 1));
    float prev_z = 0;
    for (int i = 0; i < n_per_ray; i++) {
        float t_sample = __fmaf_rn(-t_between, (float)i, 1.0f);   // contracted to one FFMA in the reference SASS
        if (randomize) {
            rng.advance((int64_t)(idx * n_per_ray));
            float rnd = rng.next_float();
            float mov = __fmaf_rn(t_between, rnd, -__fmul_rn(t_between, 0.5f));
            t_sample = __fadd_rn(t_sample, mov);
        }
        t_sample = clampf(t_sample, min_t, 1.0f);
        float z = __fdiv_rn(t_exit, t_sample);
        int s = idx * n_per_ray + i;
        s_z[s] = z;
        if (i > 0) s_dt[s - 1] = __fsub_rn(z, prev_z);
        prev_z = z;
        float px = __fmaf_rn(z, dx, ox), py = __fmaf_rn(z, dy, oy), pz = __fmaf_rn(z, dz, oz);
        if (contract) {
            float tr = t_sample * sphere_radius;
            float len = sqrtf(px * px + py * py + pz * pz);
            float f = 2 * sphere_radius - tr;
            px = f * (px / len); py = f * (py / len); pz = f * (pz / len);
        }
        s3[3 * s] = px; s3[3 * s + 1] = py; s3[3 * s + 2] = pz;
        float qx = px - cx, qy = py - cy, qz = pz - cz;
        float d2 = qx * qx + qy * qy + qz * qz;
        float inv = rsqrtf(d2);
        float dist = sqrtf(d2);
        s4[4 * s] = qx * inv; s4[4 * s + 1] = qy * inv; s4[4 * s + 2] = qz * inv;
        s4[4 * s + 3] = sphere_radius / fmaxf(1e-6f, dist);
        s_dirs[3 * s] = dx; s_dirs[3 * s + 1] = dy; s_dirs[3 * s + 2] = dz;
    }
    s_dt[idx * n_per_ray + n_per_ray - 1] = 1e10f;
    ray_fixed_dt[idx] = 0;
    start_end[2 * idx] = idx * n_per_ray;
    start_end[2 * idx + 1] = idx * n_per_ray + n_per_ray;
}

// ------------------------------------------------------------------------------------------------ Packed container
// Deterministic compaction = exclusive scan of per-ray counts + warp-per-ray coalesced copy
// (replaces the atomic slot grab + serial per-thread copy of RaySamplesPackedGPU.cuh:15-81).
constexpr int kScanThreads = 1024;
__device__ __forceinline__ int block_inclusive_scan(int v, int* smem /* 32 ints */) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    if (lane == 31) smem[w] = v;
    __syncthreads();
    if (w == 0) {
        int s = smem[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
        smem[lane] = s;
    }
    __syncthreads();
    if (w > 0) v += smem[w - 1];
    __syncthreads();
    return v;
}
// stage A: per-block scan of counts; writes exclusive offsets (block-local) and block totals
__global__ void __launch_bounds__(kScanThreads) k_scan_counts_local(int nr_rays, const int* __restrict__ start_end,
                                                                    int* __restrict__ offsets, int* __restrict__ block_sums) {
    __shared__ int sm[32];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int c = 0;
    if (i < nr_rays) { int2 se = reinterpret_cast<const int2*>(start_end)[i]; c = se.y - se.x; }
    int inc = block_inclusive_scan(c, sm);
    if (i < nr_rays) offsets[i] = inc - c;
    if (threadIdx.x == blockDim.x - 1) block_sums[blockIdx.x] = inc;
}
// stage B: one block scans the block totals in place (exclusive) and writes the grand total
__global__ void __launch_bounds__(kScanThreads) k_scan_block_sums(int nblocks, int* __restrict__ block_sums,
                                                                  int* __restrict__ total) {
    __shared__ int sm[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += blockDim.x) {
        int i = base + threadIdx.x;
        int c = i < nblocks ? block_sums[i] : 0;
        int inc = block_inclusive_scan(c, sm);
        int cr = carry;
        if (i < nblocks) block_sums[i] = cr + inc - c;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = cr + inc;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}
// stage C: warp per ray, coalesced copy of every per-sample array
__global__ void __launch_bounds__(kThreads)
k_compact_copy(int nr_rays, const float* __restrict__ pos, const float* __restrict__ pos4, const float* __restrict__ dirs,
               const float* __restrict__ z, const float* __restrict__ dt, const float* __restrict__ sdf,
               const float* __restrict__ fixed_dt, const int* __restrict__ start_end, const int* __restrict__ offsets,
               const int* __restrict__ block_sums, float* __restrict__ o_pos, float* __restrict__ o_pos4,
               float* __restrict__ o_dirs, float* __restrict__ o_z, float* __restrict__ o_dt, float* __restrict__ o_sdf,
               float* __restrict__ o_fixed_dt, int* __restrict__ o_start_end) {
    int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    int2 se = reinterpret_cast<const int2*>(start_end)[ray];
    int n = se.y - se.x;
    int os = offsets[ray] + block_sums[ray / kScanThreads];
    if (lane == 0) {
        o_fixed_dt[ray] = fixed_dt[ray];
        reinterpret_cast<int2*>(o_start_end)[ray] = make_int2(os, os + n);
    }
    for (int i = lane; i < 3 * n; i += 32) {
        o_pos[3 * os + i] = pos[3 * se.x + i];
        o_dirs[3 * os + i] = dirs[3 * se.x + i];
    }
    if (pos4) for (int i = lane; i < 4 * n; i += 32) o_pos4[4 * os + i] = pos4[4 * se.x + i];
    for (int i = lane; i < n; i += 32) {
        o_z[os + i] = z[se.x + i];
        o_dt[os + i] = dt[se.x + i];
        if (sdf) o_sdf[os + i] = sdf[se.x + i];
    }
}
// sum over rays of (end-start) -> device int (RaySamplesPacked.cu:44-55 without the host sync)
__global__ void __launch_bounds__(kScanThreads) k_count_samples(int nr_rays, const int* __restrict__ start_end,
                                                                int* __restrict__ total) {
    __shared__ int sm[32];
    int acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nr_rays; i += gridDim.x * blockDim.x) {
        int2 se = reinterpret_cast<const int2*>(start_end)[i];
        acc += se.y - se.x;
    }
    int inc = block_inclusive_scan(acc, sm);
    if (threadIdx.x == blockDim.x - 1 && inc) atomicAdd(total, inc);
}
// RaySamplesPackedGPU.cuh:84-115, warp per ray
__global__ void __launch_bounds__(kThreads) k_per_sample_ray_idx(int nr_rays, int nr_samples, const int* __restrict__ start_end,
                                                                 int* __restrict__ out) {
    int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (ray >= nr_rays) return;
    int2 se = reinterpret_cast<const int2*>(start_end)[ray];
    for (int i = se.x + lane; i < se.y; i += 32)
        if (i < nr_samples) out[i] = ray;
}

// ------------------------------------------------------------------------------------------------ SH + ray generation
// Real spherical harmonics up to degree 7 (PermutoSDFGPU.cuh:275-365). Channel c of sample i is evaluated by thread
// (i, c-group): the polynomial table is the standard one; outputs are written as a coalesced [N, degree^2] block.
template <int DEG>
__global__ void __launch_bounds__(128) k_spherical_harmonics(int n, const float* __restrict__ dirs, float* __restrict__ out) {
    constexpr int C = DEG * DEG;
    __shared__ float tile[128 * C];
    int i = blockIdx.x * 128 + threadIdx.x;
    if (i < n) {
        float v[C];
        sh_eval(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2], DEG, v);
#pragma unroll
        for (int c = 0; c < C; c++) tile[threadIdx.x * C + c] = v[c];
    }
    __syncthreads();
    long long base = (long long)blockIdx.x * 128 * C;
    int cnt = min(128, n - blockIdx.x * 128) * C;
    for (int k = threadIdx.x; k < cnt; k += 128) out[base + k] = tile[k];
}

// PermutoSDFGPU.cuh:24-127
__global__ void __launch_bounds__(kThreads)
k_random_rays_from_reel(int nr_rays, int H, int W, const float* __restrict__ rgb_reel, const float* __restrict__ mask_reel,
                        const float* __restrict__ K, const float* __restrict__ tf, const int* __restrict__ pix,
                        const int* __restrict__ img, bool has_mask, float* __restrict__ o_out, float* __restrict__ d_out,
                        float* __restrict__ gt_rgb, float* __restrict__ gt_mask) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nr_rays) return;
    int im = img[i], p = pix[i];
    float sx = (float)(p % W) + 0.5f, sy = (float)(p / W) + 0.5f;
    const float* Ki = K + 9 * im;
    const float* T = tf + 16 * im;
    float cxp = (sx - Ki[2]) / Ki[0], cyp = (sy - Ki[5]) / Ki[4];
    float tx = T[3], ty = T[7], tz = T[11];
    float wx = T[0] * cxp + T[1] * cyp + T[2] + tx;
    float wy = T[4] * cxp + T[5] * cyp + T[6] + ty;
    float wz = T[8] * cxp + T[9] * cyp + T[10] + tz;
    float vx = wx - tx, vy = wy - ty, vz = wz - tz;
    float inv = rsqrtf(vx * vx + vy * vy + vz * vz);
    int x = (int)floorf(sx), y = (int)floorf(sy);
    float m = has_mask ? mask_reel[((size_t)im * H + y) * W + x] : 1.0f;
    o_out[3 * i] = tx; o_out[3 * i + 1] = ty; o_out[3 * i + 2] = tz;
    d_out[3 * i] = vx * inv; d_out[3 * i + 1] = vy * inv; d_out[3 * i + 2] = vz * inv;
    size_t plane = (size_t)H * W;
    size_t base = (size_t)im * 3 * plane + (size_t)y * W + x;
    gt_rgb[3 * i] = rgb_reel[base] * m;
    gt_rgb[3 * i + 1] = rgb_reel[base + plane] * m;
    gt_rgb[3 * i + 2] = rgb_reel[base + 2 * plane] * m;
    gt_mask[i] = m;
}

inline GridGeom geom(int V, float extent, const float* t) {
    GridGeom g;
    g.V = V; g.extent = extent; g.tx = t[0]; g.ty = t[1]; g.tz = t[2];
    int ex = 0;
    float m = frexpf(extent, &ex);
    g.inv_extent = (m == 0.5f) ? 1.0f / extent : 0.0f;      // exact reciprocal only for powers of two
    g.inv_V = 1.0f / (float)V;
    return g;
}
#define ST ((cudaStream_t)stream)
}  // namespace

// =================================================================================================== C ABI
extern "C" {

int psdf_sphere_ray_intersection(int nr_rays, float radius, const float center[3], const float* origins, const float* dirs,
                                 float* pts_entry, float* t_entry, float* pts_exit, float* t_exit, uint8_t* hit, void* stream) {
    if (nr_rays < 0) return PSDF_ERR_ARG;
    if (nr_rays == 0) return PSDF_OK;
    k_sphere_ray_intersection<<<div_up(nr_rays, kThreads), kThreads, 0, ST>>>(nr_rays, radius, center[0], center[1], center[2],
                                                                             origins, dirs, pts_entry, t_entry, pts_exit,
                                                                             t_exit, hit);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_sphere_rand_points_inside(int n, float radius, const float* phi, const float* costheta, const float* u, float* points,
                                   void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_sphere_rand_points<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, radius, phi, costheta, u, points);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_sphere_check_point_inside(int n, float radius, const float center[3], const float* points, uint8_t* out, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_sphere_inside<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, radius, center[0], center[1], center[2], points, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_occ_compute_grid_points(int n, int V, float extent, const float trans[3], const int* idx, uint64_t rng_state,
                                 uint64_t rng_inc, int randomize, float* out, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_occ_grid_points<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, geom(V, extent, trans), idx, Pcg32(rng_state, rng_inc),
                                                               randomize != 0, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_occ_update_with_density(int n, const float* density, const int* idx, float decay, float thresh, float* values,
                                 uint8_t* occ, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    // deterministic mode: arbitration of repeated voxels (indices must stay below the grid size reserved by psdf_set_deterministic)
    const DetBufs* dbuf = det_buffers();
    int* winner = (dbuf && idx) ? dbuf->winner : nullptr;
    if (winner) k_occ_claim<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, idx, winner, dbuf->voxels);
    k_occ_update_density<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, density, idx, decay, thresh, values, occ, winner, winner ? dbuf->voxels : 0);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_occ_update_with_sdf(int n, const float* sdf, const int* idx, float extent, int V, float inv_s, const float* inv_s_dev,
                             float thresh, int random_sample_variant, float* values, uint8_t* occ, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    const DetBufs* dbuf = det_buffers();
    int* winner = (dbuf && idx) ? dbuf->winner : nullptr;
    if (winner && (long long)V * V * V > dbuf->voxels) return PSDF_ERR_UNSUPPORTED;   // reserve more with psdf_set_deterministic
    if (winner) k_occ_claim<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, idx, winner, dbuf->voxels);
    // error range of the sdf inside a voxel: 1.3 (full grid, :437) or 1.0 (random subset, :497) half diagonals
    float voxel = extent / (float)V;
    float half = (float)((double)voxel / 2.0);
    float half_diag = sqrtf(3.0f) * half;
    float range = random_sample_variant ? (float)(1.0 * (double)half_diag) : (float)(1.3 * (double)half_diag);
    k_occ_update_sdf<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, sdf, idx, range, inv_s, inv_s_dev, thresh, values, occ, winner, winner ? dbuf->voxels : 0);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_occ_check_occupancy(int n, int V, float extent, const float trans[3], const uint8_t* occ, const float* points,
                             uint8_t* out, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_occ_check<<<div_up(n, kThreads), kThreads, 0, ST>>>(n, geom(V, extent, trans), occ, points, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_occ_compute_samples_in_occupied_regions(int nr_rays, int V, float extent, const float trans[3], const float* origins,
                                                 const float* dirs, const float* t_entry, const float* t_exit,
                                                 const uint8_t* occ, float min_dist, int max_per_ray, int max_nr_samples,
                                                 uint64_t rng_state, uint64_t rng_inc, int jitter, int slot_mode,
                                                 float* s_pos, float* s_dirs, float* s_z, float* s_dt, float* ray_fixed_dt,
                                                 int* ray_start_end, int* cur_nr_samples, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    if (slot_mode == 1 && (long long)nr_rays * max_per_ray > (long long)max_nr_samples) return PSDF_ERR_ARG;
    const GridGeom gg = geom(V, extent, trans);
    auto kern = gg.inv_extent != 0.0f ? k_occ_samples_in_occupied<true> : k_occ_samples_in_occupied<false>;
    kern<<<div_up(nr_rays, kOccWarpsPerBlock), kOccWarpsPerBlock * 32, 0, ST>>>(nr_rays, gg, origins, dirs, t_entry, t_exit,
                                                                 occ, min_dist, max_per_ray, max_nr_samples,
                                                                 Pcg32(rng_state, rng_inc), jitter != 0, slot_mode, s_pos,
                                                                 s_dirs, s_z, s_dt, ray_fixed_dt, ray_start_end,
                                                                 cur_nr_samples);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_occ_compute_first_sample_start(int nr_rays, int V, float extent, const float trans[3], const float* origins,
                                        const float* dirs, const float* t_entry, const float* t_exit, const uint8_t* occ,
                                        int max_nr_samples, int slot_mode, float* s_pos, float* s_dirs, float* s_z, float* s_dt,
                                        float* ray_fixed_dt, int* ray_start_end, int* cur_nr_samples, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    if (slot_mode == 1 && nr_rays > max_nr_samples) return PSDF_ERR_ARG;
    k_occ_first_sample<<<div_up(nr_rays, 128), 128, 0, ST>>>(nr_rays, geom(V, extent, trans), origins, dirs, t_entry, t_exit, occ,
                                                            max_nr_samples, slot_mode, s_pos, s_dirs, s_z, s_dt, ray_fixed_dt,
                                                            ray_start_end, cur_nr_samples);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_occ_advance_sample_to_next_occupied_voxel(int n, int V, float extent, const float trans[3], const float* dirs,
                                                   float* pos_io, const uint8_t* occ, uint8_t* within, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_occ_advance_to_next_occupied<<<div_up(n, 128), 128, 0, ST>>>(n, geom(V, extent, trans), dirs, pos_io, occ, within);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_sampler_fg(int nr_rays, const float* origins, const float* dirs, const float* t_entry, const float* t_exit,
                    float min_dist, int max_per_ray, int max_nr_samples, uint64_t rng_state, uint64_t rng_inc, int jitter,
                    int slot_mode, float* s_pos, float* s_dirs, float* s_z, float* s_dt, float* ray_fixed_dt,
                    int* ray_start_end, int* cur_nr_samples, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    if (slot_mode == 1 && (long long)nr_rays * max_per_ray > (long long)max_nr_samples) return PSDF_ERR_ARG;
    k_sampler_fg<<<div_up(nr_rays, 64), 64, 0, ST>>>(nr_rays, origins, dirs, t_entry, t_exit, min_dist, max_per_ray,
                                                    max_nr_samples, Pcg32(rng_state, rng_inc), jitter != 0, slot_mode, s_pos,
                                                    s_dirs, s_z, s_dt, ray_fixed_dt, ray_start_end, cur_nr_samples);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_sampler_bg(int nr_rays, int n_per_ray, const float* origins, const float* dirs, const float* t_exit,
                    float sphere_radius, const float sphere_center[3], uint64_t rng_state, uint64_t rng_inc, int randomize,
                    int contract, float* s3, float* s4, float* s_dirs, float* s_z, float* s_dt, float* ray_fixed_dt,
                    int* ray_start_end, void* stream) {
    if (nr_rays <= 0 || n_per_ray < 2) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_sampler_bg<<<div_up(nr_rays, 64), 64, 0, ST>>>(nr_rays, n_per_ray, origins, dirs, t_exit, sphere_radius, sphere_center[0],
                                                    sphere_center[1], sphere_center[2], Pcg32(rng_state, rng_inc),
                                                    randomize != 0, contract != 0, s3, s4, s_dirs, s_z, s_dt, ray_fixed_dt,
                                                    ray_start_end);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_rng_advance_dev(uint64_t* rng_dev, long long delta, void* stream) {
    if (!rng_dev || delta < 0) return PSDF_ERR_ARG;
    k_rng_advance<<<1, 1, 0, ST>>>(rng_dev, delta);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

long long psdf_packed_compact_workspace_bytes(int nr_rays) {
    int nblocks = div_up(nr_rays > 0 ? nr_rays : 1, kScanThreads);
    return (long long)sizeof(int) * ((long long)nr_rays + nblocks + 1);
}
int psdf_packed_count_samples(int nr_rays, const int* ray_start_end, int* total_dev, void* stream) {
    cudaMemsetAsync(total_dev, 0, sizeof(int), ST);
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    int blocks = min(div_up(nr_rays, kScanThreads), 132);
    k_count_samples<<<blocks, kScanThreads, 0, ST>>>(nr_rays, ray_start_end, total_dev);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
// workspace layout: [offsets: nr_rays][block_sums: nblocks][total: 1]; total is also the device count after the call
int psdf_packed_compact_scan(int nr_rays, const int* ray_start_end, int* workspace, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    int nblocks = div_up(nr_rays, kScanThreads);
    int* offsets = workspace;
    int* block_sums = workspace + nr_rays;
    int* total = block_sums + nblocks;
    k_scan_counts_local<<<nblocks, kScanThreads, 0, ST>>>(nr_rays, ray_start_end, offsets, block_sums);
    k_scan_block_sums<<<1, kScanThreads, 0, ST>>>(nblocks, block_sums, total);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_packed_compact_copy(int nr_rays, const float* pos, const float* pos4, const float* dirs, const float* z,
                             const float* dt, const float* sdf, const float* fixed_dt, const int* ray_start_end,
                             const int* workspace, float* o_pos, float* o_pos4, float* o_dirs, float* o_z, float* o_dt,
                             float* o_sdf, float* o_fixed_dt, int* o_start_end, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    const int* offsets = workspace;
    const int* block_sums = workspace + nr_rays;
    k_compact_copy<<<div_up((long long)nr_rays * 32, kThreads), kThreads, 0, ST>>>(nr_rays, pos, pos4, dirs, z, dt, sdf, fixed_dt,
                                                                                  ray_start_end, offsets, block_sums, o_pos,
                                                                                  o_pos4, o_dirs, o_z, o_dt, o_sdf, o_fixed_dt,
                                                                                  o_start_end);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_packed_per_sample_ray_idx(int nr_rays, int nr_samples, const int* ray_start_end, int* out, void* stream) {
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_per_sample_ray_idx<<<div_up((long long)nr_rays * 32, kThreads), kThreads, 0, ST>>>(nr_rays, nr_samples, ray_start_end, out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_spherical_harmonics(int n, int degree, const float* dirs, float* out, void* stream) {
    if (n <= 0) return n == 0 ? PSDF_OK : PSDF_ERR_ARG;
    int blocks = div_up(n, 128);
    switch (degree) {
        case 1: k_spherical_harmonics<1><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        case 2: k_spherical_harmonics<2><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        case 3: k_spherical_harmonics<3><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        case 4: k_spherical_harmonics<4><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        case 5: k_spherical_harmonics<5><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        case 6: k_spherical_harmonics<6><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        case 7: k_spherical_harmonics<7><<<blocks, 128, 0, ST>>>(n, dirs, out); break;
        default: return PSDF_ERR_ARG;
    }
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}
int psdf_random_rays_from_reel(int nr_rays, int nr_images, int H, int W, const float* rgb_reel, const float* mask_reel,
                               const float* K, const float* tf_world_cam, const int* pixel_indices, const int* img_indices,
                               int has_mask, float* origins, float* dirs, float* gt_rgb, float* gt_mask, void* stream) {
    (void)nr_images;
    if (nr_rays <= 0) return nr_rays == 0 ? PSDF_OK : PSDF_ERR_ARG;
    k_random_rays_from_reel<<<div_up(nr_rays, kThreads), kThreads, 0, ST>>>(nr_rays, H, W, rgb_reel, mask_reel, K, tf_world_cam,
                                                                           pixel_indices, img_indices, has_mask != 0, origins,
                                                                           dirs, gt_rgb, gt_mask);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
