/*
 * psdf_b200.h -- C ABI of libpsdf_b200.so, the sm_90a (H100) implementation of PermutoSDF's per-ray
 * training / sphere-tracing hot path.
 *
 * Boundary: the reference exposes this path to Python as a pybind11 module `permuto_sdf`
 * (src/PyBridge.cxx:30-169) plus the external package `permutohedral_encoding`
 * (permuto_sdf_py/models/models.py:20,149,186). Both are re-created in Python on top of THIS header
 * (permuto_sdf_b200/permuto_sdf, permuto_sdf_b200/permutohedral_encoding); every entry point below names
 * the reference method it replaces. INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *   - all pointers are DEVICE pointers (contiguous, fp32 / int32 / uint8 bool) unless the name ends in
 *     `[3]` or `[6]` (small host arrays passed by the caller); no allocation happens inside the library;
 *   - `stream` is a cudaStream_t; kernels are asynchronous on it; the library never synchronises;
 *   - return value: 0 = ok, <0 = error (PSDF_ERR_*); no global state: RNG state is passed explicitly
 *     as the (state, inc) pair of a pcg32 generator (kernels/permuto_sdf/pcg32.h:45-171). rng_inc == 0 (never a
 *     valid pcg32 stream) marks rng_state as a DEVICE pointer to uint64_t[2] = {state, inc}: the generator then lives
 *     in device memory, is advanced with psdf_rng_advance_dev, and the call can be replayed from a CUDA graph;
 *   - packed ray containers follow RaySamplesPacked (include/permuto_sdf/RaySamplesPacked.cuh:7-46):
 *     ray_start_end is int32 [R,2] = [start,end); `equal`/`fixed_n` is the rays_have_equal_nr_of_samples
 *     fast path; rays with end > max_nr_samples or zero samples are skipped
 *     (kernels/permuto_sdf/VolumeRenderingGPU.cuh:30-60,103).
 */
#ifndef PSDF_B200_H
#define PSDF_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* changes when an existing entry point changes its signature or behaviour; entry points that are only added leave it as it is */
#define PSDF_ABI_VERSION 2
#define PSDF_ERR_ARG_ -1
#define PSDF_ERR_LAUNCH_ -2
#define PSDF_ERR_UNSUPPORTED_ -3

int psdf_abi_version(void);
/* 1 when a compute-capability 9.x (H100, the library's sm_90a target) device is present, else 0 (never a CPU fallback) */
int psdf_device_ok(void);
/* Deterministic mode of the current device. Off (the default): gradient reductions use float atomics, so a training step's
 * gradients differ from run to run in their last bits. On: the training path's reductions (fused SDF / colour backward, compositing
 * backward, Lipschitz backward, loss terms) accumulate in 64-bit fixed point (2^-34 grid, |values| < 5.3e8) and a random occupancy
 * update lets the last sample of a repeated voxel win, so runs with the same inputs give the same bits. lattice_entries = the
 * largest L * T * F of a backward call, voxels = the largest occupancy grid (larger calls return PSDF_ERR_UNSUPPORTED). Allocates or
 * frees device memory: call outside CUDA-graph capture with no launch of this library in flight.
 * Launches of one fused kernel must not run concurrently on a device: each fused kernel keeps its accumulators in one per-device
 * area (and, in deterministic mode, shares the fixed-point accumulators). */
int psdf_set_deterministic(int on, long long lattice_entries, long long voxels);

/* ---------------------------------------------------------------- Sphere (include/permuto_sdf/Sphere.cuh:12-24) */
/* Sphere::ray_intersection, src/Sphere.cu:42-79 */
int psdf_sphere_ray_intersection(int nr_rays, float radius, const float center[3], const float* origins, const float* dirs,
                                 float* pts_entry, float* t_entry, float* pts_exit, float* t_exit, uint8_t* hit, void* stream);
/* Sphere::rand_points_inside, src/Sphere.cu:82-109 (random inputs phi,costheta,u are drawn by the caller) */
int psdf_sphere_rand_points_inside(int n, float radius, const float* phi, const float* costheta, const float* u, float* points,
                                   void* stream);
/* Sphere::check_point_inside_primitive, src/Sphere.cu:111-119 */
int psdf_sphere_check_point_inside(int n, float radius, const float center[3], const float* points, uint8_t* out, void* stream);

/* ---------------------------------------------------------------- AABB (permuto_sdf_py/utils/aabb.py:7-114) */
/* AABB.ray_intersection, aabb.py:47-100, bit-identical to its torch ops: box of sizes[3] centred at translation[3]; -> entry points
 * [N,3] and t [N], exit points [N,3] and t [N], hit [N] (misses: t = 0 at both ends); t_entry is clamped at 0 */
int psdf_aabb_ray_intersection(int nr_rays, const float sizes[3], const float translation[3], const float* origins, const float* dirs,
                               float* pts_entry, float* t_entry, float* pts_exit, float* t_exit, uint8_t* hit, void* stream);

/* ---------------------------------------------------------------- OccupancyGrid (include/permuto_sdf/OccupancyGrid.cuh:19-64) */
/* compute_grid_points (idx==NULL, n==V^3) / compute_random_sample_of_grid_points (idx = chosen voxels),
 * src/OccupancyGrid.cu:88-117,179-208 */
int psdf_occ_compute_grid_points(int n, int V, float extent, const float trans[3], const int* idx, uint64_t rng_state,
                                 uint64_t rng_inc, int randomize, float* out, void* stream);
/* update_with_density (idx==NULL) / update_with_density_random_sample, src/OccupancyGrid.cu:368-420 */
int psdf_occ_update_with_density(int n, const float* density, const int* idx, float decay, float thresh, float* values,
                                 uint8_t* occ, void* stream);
/* update_with_sdf (idx==NULL, scalar inv_s, variant 0) / update_with_sdf_random_sample (inv_s_dev = 1-element
 * device tensor, variant 1), src/OccupancyGrid.cu:422-475 */
int psdf_occ_update_with_sdf(int n, const float* sdf, const int* idx, float extent, int V, float inv_s, const float* inv_s_dev,
                             float thresh, int random_sample_variant, float* values, uint8_t* occ, void* stream);
/* check_occupancy, src/OccupancyGrid.cu:339-365 */
int psdf_occ_check_occupancy(int n, int V, float extent, const float trans[3], const uint8_t* occ, const float* points,
                             uint8_t* out, void* stream);
/* compute_samples_in_occupied_regions, src/OccupancyGrid.cu:212-257.
 * slot_mode 1: ray i owns slots [i*max_per_ray, ...) (deterministic, needs nr_rays*max_per_ray <= max_nr_samples);
 * slot_mode 0: slots from a global atomic counter like the reference. cur_nr_samples must be zeroed by the caller. */
int psdf_occ_compute_samples_in_occupied_regions(int nr_rays, int V, float extent, const float trans[3], const float* origins,
                                                 const float* dirs, const float* t_entry, const float* t_exit,
                                                 const uint8_t* occ, float min_dist, int max_per_ray, int max_nr_samples,
                                                 uint64_t rng_state, uint64_t rng_inc, int jitter, int slot_mode,
                                                 float* s_pos, float* s_dirs, float* s_z, float* s_dt, float* ray_fixed_dt,
                                                 int* ray_start_end, int* cur_nr_samples, void* stream);
/* compute_first_sample_start_of_occupied_regions, src/OccupancyGrid.cu:259-300 */
int psdf_occ_compute_first_sample_start(int nr_rays, int V, float extent, const float trans[3], const float* origins,
                                        const float* dirs, const float* t_entry, const float* t_exit, const uint8_t* occ,
                                        int max_nr_samples, int slot_mode, float* s_pos, float* s_dirs, float* s_z, float* s_dt,
                                        float* ray_fixed_dt, int* ray_start_end, int* cur_nr_samples, void* stream);
/* advance_sample_to_next_occupied_voxel, src/OccupancyGrid.cu:302-337 (pos updated in place, like the reference) */
int psdf_occ_advance_sample_to_next_occupied_voxel(int n, int V, float extent, const float trans[3], const float* dirs,
                                                   float* pos_io, const uint8_t* occ, uint8_t* within, void* stream);

/* ---------------------------------------------------------------- RaySampler (include/permuto_sdf/RaySampler.cuh:21-22) */
int psdf_sampler_fg(int nr_rays, const float* origins, const float* dirs, const float* t_entry, const float* t_exit,
                    float min_dist, int max_per_ray, int max_nr_samples, uint64_t rng_state, uint64_t rng_inc, int jitter,
                    int slot_mode, float* s_pos, float* s_dirs, float* s_z, float* s_dt, float* ray_fixed_dt,
                    int* ray_start_end, int* cur_nr_samples, void* stream);
int psdf_sampler_bg(int nr_rays, int n_per_ray, const float* origins, const float* dirs, const float* t_exit,
                    float sphere_radius, const float sphere_center[3], uint64_t rng_state, uint64_t rng_inc, int randomize,
                    int contract, float* s3, float* s4, float* s_dirs, float* s_z, float* s_dt, float* ray_fixed_dt,
                    int* ray_start_end, void* stream);

/* device-resident generator: state <- state advanced by `delta` draws (the reference advances its static generators by 2^32
 * after every jittered call, e.g. src/OccupancyGrid.cu:254) */
int psdf_rng_advance_dev(uint64_t* rng_dev, long long delta, void* stream);

/* ---------------------------------------------------------------- RaySamplesPacked (src/RaySamplesPacked.cu:44-146) */
long long psdf_packed_compact_workspace_bytes(int nr_rays);
/* compute_exact_nr_samples without the host sync: total_dev <- sum(end-start) */
int psdf_packed_count_samples(int nr_rays, const int* ray_start_end, int* total_dev, void* stream);
/* compact_to_valid_samples = scan (fills workspace; workspace[nr_rays + nblocks] is the total) + copy */
int psdf_packed_compact_scan(int nr_rays, const int* ray_start_end, int* workspace, void* stream);
int psdf_packed_compact_copy(int nr_rays, const float* pos, const float* pos4, const float* dirs, const float* z,
                             const float* dt, const float* sdf, const float* fixed_dt, const int* ray_start_end,
                             const int* workspace, float* o_pos, float* o_pos4, float* o_dirs, float* o_z, float* o_dt,
                             float* o_sdf, float* o_fixed_dt, int* o_start_end, void* stream);
/* compute_per_sample_ray_idx */
int psdf_packed_per_sample_ray_idx(int nr_rays, int nr_samples, const int* ray_start_end, int* out, void* stream);

/* ---------------------------------------------------------------- VolumeRendering (include/permuto_sdf/VolumeRendering.cuh:22-38) */
#define PSDF_RSP int nr_rays, int max_nr_samples, const int* ray_start_end, int equal, int fixed_n
/* A ray is skipped when it is empty or its end > max_nr_samples. Of a skipped ray's outputs only these rows are written:
 * bg_transmittance = 1 (cumprod), out = 0 (integrate), sum_ray = 0 (sum), pred_rgb = 0, pred_depth = 0, bg_transmittance = 1 (NeRF
 * render) and its importance samples (pos = dirs = 0, z = -1). The NeRF render and its backward stop a ray once T < 1e-4: the
 * per-sample rows after that point are not written. */
int psdf_vr_cumprod_alpha2transmittance(PSDF_RSP, const float* one_minus_alpha, float* transmittance, float* bg_transmittance, void* stream);
int psdf_vr_integrate_with_weights(PSDF_RSP, const float* vals, const float* weights, float* out, void* stream);
int psdf_vr_sdf2alpha(PSDF_RSP, const float* ray_fixed_dt, const float* samples_dt, const float* sdf, float inv_s, int dynamic_inv_s,
                      float inv_s_multiplier, float* alpha, void* stream);
int psdf_vr_sum_over_each_ray(PSDF_RSP, int val_dim, const float* vals, float* sum_ray, float* sum_sample, void* stream);
int psdf_vr_cumsum_over_each_ray(PSDF_RSP, const float* vals, int inverse, float* out, void* stream);
int psdf_vr_compute_cdf(PSDF_RSP, const float* weights, float* cdf, void* stream);
int psdf_vr_importance_sample(PSDF_RSP, const float* origins, const float* dirs, const float* ray_fixed_dt, const float* samples_z,
                              const float* cdf, int nr_imp, uint64_t rng_state, uint64_t rng_inc, int jitter, float* o_pos,
                              float* o_dirs, float* o_z, void* stream);
/* (importance_sample / importance_round) a ray with a single sample has no cdf interval to draw from: its importance samples are
 * those of a skipped ray. Every other output of a ray depends on that ray's rows only. */
long long psdf_vr_combine_workspace_bytes(int nr_rays);
/* one round of importance_sampling_sdf_model (permuto_sdf_py/utils/sdf_utils.py): sdf2alpha -> clip -> cumprod(1 - alpha + 1e-7) ->
 * weights -> per-ray normalisation (clamp 1e-6) -> cdf -> importance_sample, one launch, bit-identical to the separate calls.
 * cdf [N] is scratch + output (the per-ray exclusive cdf). */
int psdf_vr_importance_round(PSDF_RSP, const float* origins, const float* dirs, const float* ray_fixed_dt, const float* samples_dt,
                             const float* samples_z, const float* sdf, float inv_s, int dynamic_inv_s, float inv_s_multiplier, int nr_imp,
                             uint64_t rng_state, uint64_t rng_inc, int jitter, float* cdf, float* o_pos, float* o_dirs, float* o_z,
                             void* stream);
/* merge of each ray's uniform and importance samples by z (the uniform one first only if strictly smaller), into slots scanned in
 * ray order; rays with at most one uniform sample get start_end (0, 0) and fixed_dt 0. Any merged length is supported. */
int psdf_vr_combine_uniform_samples_with_imp(PSDF_RSP, const float* origins, const float* dirs, const float* t_exit,
                                             const float* u_fixed_dt, const float* u_z, const float* u_sdf, int u_has_sdf,
                                             int imp_n, const float* i_z, const float* i_sdf, int i_has_sdf, int c_max,
                                             int* workspace, float* c_pos, float* c_dirs, float* c_z, float* c_dt, float* c_sdf,
                                             float* c_fixed_dt, int* c_start_end, void* stream);
int psdf_vr_cumprod_alpha2transmittance_backward(PSDF_RSP, const float* grad_bg_transmittance, const float* alpha,
                                                 const float* bg_transmittance, const float* cumsumLV, float* grad_alpha,
                                                 void* stream);
int psdf_vr_integrate_with_weights_backward(PSDF_RSP, const float* grad_pred, const float* vals, const float* weights,
                                            int reference_bug, float* grad_vals, float* grad_weights, void* stream);
int psdf_vr_sum_over_each_ray_backward(PSDF_RSP, int val_dim, const float* grad_sum_ray, const float* grad_sum_sample,
                                       float* grad_vals, void* stream);
int psdf_vr_compute_dt(PSDF_RSP, int use_t_exit, const float* t_exit, const float* samples_z, float* dt, void* stream);
int psdf_vr_volume_render_nerf(PSDF_RSP, const float* rgb, const float* radiance, const float* samples_z, const float* samples_dt,
                               float* pred_rgb, float* pred_depth, float* bg_transmittance, float* weight_per_sample, void* stream);
int psdf_vr_volume_render_nerf_backward(PSDF_RSP, const float* grad_pred_rgb, const float* grad_bg_transmittance,
                                        const float* pred_rgb, const float* bg_transmittance, const float* rgb,
                                        const float* radiance, const float* samples_dt, float* grad_rgb, float* grad_radiance,
                                        void* stream);

/* Fused NeuS compositing + per-ray losses (training): replaces VolumeRenderingNeus.compute_weights + integrate
 * (permuto_sdf_py/volume_rendering/volume_rendering_modules.py:129-176) and the rgb / mask / eikonal losses
 * (permuto_sdf_py/train_permuto_sdf.py:349-383, permuto_sdf_py/utils/permuto_sdf_utils.py:43-51) in one launch each way.
 * sdf [N], grad/rgb/dirs [N,3], dt [N], inv_s_dev [1] (device scalar, clipped to [1e-6,1e6] inside), gt_rgb [R,3],
 * gt_mask [R] or NULL, hit [R] u8 or NULL, bg_rgb [R,3] or NULL (pred += bg_T * bg_rgb).
 * ray_loss [R,3] = {sum_c |gt-pred| * hit, BCE(clip(w_sum,1e-3,1-1e-3), mask), sum_i (|grad_i|-1)^2}. */
int psdf_neus_render_loss_forward(PSDF_RSP, const float* sdf, const float* grad, const float* rgb, const float* dirs, const float* dt,
                                  const float* inv_s_dev, float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb,
                                  const float* gt_mask, const uint8_t* hit, const float* bg_rgb, float* alpha, float* transmittance, float* weights,
                                  float* pred_rgb, float* weights_sum, float* bg_transmittance, float* ray_loss, void* stream);
/* d loss / d {sdf, grad, rgb, bg_rgb, inv_s} for loss = g_total * (scale_rgb * sum rgb-term + scale_mask * sum bce + scale_eik * sum eik);
 * g_total_dev [1] device scalar or NULL (=1); g_bg_rgb / g_inv_s may be NULL; g_inv_s is accumulated (+=).
 * cos_anneal_dev [1] (both calls) overrides cos_anneal_ratio when not NULL; nr_samples_dev [1] int, when not NULL, divides
 * scale_eik on the device (static-capacity containers under CUDA-graph replay, where the sample count is not known on the host). */
int psdf_neus_render_loss_backward(PSDF_RSP, const float* sdf, const float* grad, const float* rgb, const float* dirs, const float* dt,
                                   const float* inv_s_dev, float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb,
                                   const float* gt_mask, const uint8_t* hit, const float* bg_rgb, const float* alpha, const float* transmittance,
                                   const float* pred_rgb, const float* weights_sum, const float* bg_transmittance,
                                   const float* g_total_dev, float scale_rgb, float scale_mask, float scale_eik,
                                   const int* nr_samples_dev, float* g_sdf,
                                   float* g_grad, float* g_rgb, float* g_bg_rgb, float* g_inv_s, void* stream);

/* ---------------------------------------------------------------- colour network helpers
 * LipshitzMLP weight normalisation (permuto_sdf_py/models/models.py:96-110): W_eff[r,:] = W[r,:] * min(1, softplus(c) / sum|W[r,:]|);
 * W [rows,cols], c [1] device scalar. Backward: grad_W (=), grad_c (+=, may be NULL). */
int psdf_lipschitz_normalize(int rows, int cols, const float* W, const float* c, float* W_eff, void* stream);
int psdf_lipschitz_normalize_backward(int rows, int cols, const float* W, const float* c, const float* grad_W_eff, float* grad_W,
                                      float* grad_c, void* stream);
/* Colorcal.calib_RGB_samples_packed + sigmoid (models.py:395-414, 677-741) on packed samples: out = sigmoid(x (1 + weight_delta[img]) +
 * bias[img]), identity calibration for img == fixed_img or img_idx == NULL (img_idx [R] per ray). Rows outside every ray are not
 * written. Backward: grad_x (=, rows inside rays), grad_weight_delta / grad_bias [nr_imgs,3] (+=, may be NULL). */
int psdf_calib_sigmoid_forward(PSDF_RSP, const float* x, const int* img_idx, const float* weight_delta, const float* bias, int fixed_img,
                               float* out, void* stream);
int psdf_calib_sigmoid_backward(PSDF_RSP, const float* x, const float* out, const float* grad_out, const int* img_idx,
                                const float* weight_delta, int fixed_img, float* grad_x, float* grad_weight_delta, float* grad_bias,
                                void* stream);

/* Curvature loss of SDF.get_sdf_and_curvature_1d_precomputed_gradient_normal_based (models.py:261-294): shifted sample positions
 * points + eps * cross(normalize(sdf_grad), normalize(rand_dirs)); curvature [n] = acos(clamp(n . n_shifted)) / pi (rows >=
 * nr_valid_dev[0] give 0; nr_valid_dev may be NULL) with loss_sum [1] += their sum; backward of  g_loss * scale * mean-or-sum:
 * the sum is divided by max(nr_valid, 1) when nr_valid_dev is given. */
int psdf_curvature_shift_points(int n, const float* points, const float* sdf_grad, const float* rand_dirs, float eps, float* out,
                                void* stream);
int psdf_curvature_loss_forward(int n, const float* sdf_grad, const float* sdf_grad_shifted, const int* nr_valid_dev, float* curvature,
                                float* loss_sum, void* stream);
int psdf_curvature_loss_backward(int n, const float* sdf_grad, const float* sdf_grad_shifted, const int* nr_valid_dev,
                                 const float* g_loss_dev, float scale, float* grad_sdf_grad, float* grad_sdf_grad_shifted, void* stream);

/* ---------------------------------------------------------------- PermutoSDF statics (include/permuto_sdf/PermutoSDF.cuh:46-55) */
int psdf_spherical_harmonics(int n, int degree, const float* dirs, float* out, void* stream);
int psdf_random_rays_from_reel(int nr_rays, int nr_images, int H, int W, const float* rgb_reel, const float* mask_reel,
                               const float* K, const float* tf_world_cam, const int* pixel_indices, const int* img_indices,
                               int has_mask, float* origins, float* dirs, float* gt_rgb, float* gt_mask, void* stream);

/* ---------------------------------------------------------------- permutohedral_encoding (external package; call sites
 * permuto_sdf_py/models/models.py:149,186; semantics SURVEY.md Appendix B)
 * pos [N,D] fp32, lattice [L,T,F] fp32, scale_factor [L,D], shift [L,D], window [L];
 * out [N,(L+E)*F] with E=ceil(D/F) concat columns (the D coordinates * points_scaling, then zeros) when concat_points.
 * Supported: D in {2, 3, 4, 5, 6}, F in {1, 2, 4, 8}, 1 <= L <= 32, T >= 1; any other shape returns PSDF_ERR_UNSUPPORTED before the
 * device is touched. lattice (and grad_lattice) must be F*4-byte aligned, 16-byte for F >= 4 (else PSDF_ERR_ARG). The five entry
 * points below share this contract. */
int psdf_enc_forward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                     const float* shift, const float* window, int concat_points, float points_scaling, float* out, void* stream);
/* grad wrt lattice (+=, caller zeroes) and/or positions (=) from grad_out [N,(L+E)*F]; either output may be NULL */
int psdf_enc_backward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                      const float* shift, const float* window, int concat_points, float points_scaling, const float* grad_out,
                      float* grad_lattice, float* grad_pos, void* stream);
/* double backward from the positions gradient: given gg_pos [N,D] (grad of grad_pos) produce
 * grad_lattice (+=) and grad_grad_out [N,(L+E)*F] (=); either may be NULL */
int psdf_enc_double_backward(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                             const float* shift, const float* window, int concat_points, float points_scaling,
                             const float* gg_pos, const float* grad_out, float* grad_lattice, float* grad_grad_out, void* stream);
/* Deterministic twins of psdf_enc_backward and psdf_enc_double_backward: the same outputs, except that the lattice gradient is
 * reduced in 64-bit fixed point (2^-34 grid, the unit of psdf_set_deterministic). Every contribution is rounded to the grid before
 * anything is added to it, so grad_lattice depends only on the multiset of (pos, grad_out[, gg_pos]) rows, not on their order or the
 * run. grad_pos and grad_grad_out are bit-identical to the float entry points'. fx_lattice: caller-owned [L,T,F] accumulators, 8-byte
 * aligned, zero on entry and zero again on return (the totals are added to grad_lattice, +=, and cleared); the library never
 * allocates. grad_lattice NULL: exactly the float entry point, fx_lattice ignored. grad_lattice without fx_lattice: PSDF_ERR_ARG. */
int psdf_enc_backward_fx(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                         const float* shift, const float* window, int concat_points, float points_scaling, const float* grad_out,
                         float* grad_lattice, float* grad_pos, uint64_t* fx_lattice, void* stream);
int psdf_enc_double_backward_fx(int N, int D, int L, int F, int T, const float* pos, const float* lattice, const float* scale_factor,
                                const float* shift, const float* window, int concat_points, float points_scaling,
                                const float* gg_pos, const float* grad_out, float* grad_lattice, float* grad_grad_out,
                                uint64_t* fx_lattice, void* stream);

/* ---------------------------------------------------------------- fused encoding + SDF MLP (wgmma)
 * Replaces SDF.forward / SDF.get_sdf_and_gradient of permuto_sdf_py/models/models.py:176-259 for evaluations that
 * need no parameter gradients: importance sampling (sdf_utils.py:388,401), occupancy refresh
 * (train_permuto_sdf.py:388-391), sphere tracing (sdf_utils.py:166,199-204).
 * MLP = Linear(in,h) GELU Linear(h,h) GELU Linear(h,h) GELU Linear(h,out), weights in torch.nn.Linear layout.
 * psdf_sdf_mlp_pack converts them once per weight update into the tensor-core operand blob. */
long long psdf_sdf_mlp_blob_bytes(int in_dim, int hidden, int out_dim);
int psdf_sdf_mlp_pack(int in_dim, int hidden, int out_dim, const float* W0, const float* b0, const float* W1, const float* b1,
                      const float* W2, const float* b2, const float* W3, const float* b3, uint8_t* blob, void* stream);
/* pos [N,3] -> sdf [N], grad [N,3] (NULL: value only), geom [N,out_dim-1] (NULL: skip). D = 3, F = 2, L % 4 == 0,
 * concat_points on (in_dim = 2L + 4). */
int psdf_sdf_fused_forward(int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor, const float* shift,
                           const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, float* sdf,
                           float* grad, float* geom, void* stream);
/* Fused sphere tracing (sphere_trace, permuto_sdf_py/utils/sdf_utils.py:120-218): nr_iters iterations of
 *   sdf = SDF(p); p += dir * sdf * sdf_multiplier; converged |= |sdf| < tresh | left the occupied region / bounding sphere
 * with advance_sample_to_next_occupied_voxel applied after every step when an occupancy grid is given (occupancy != NULL; else
 * the bounding-sphere test). Persistent CTAs of 128 ray slots pull rays from a global queue and refill finished slots;
 * pos [N,3] start points, dirs [N,3]; pos_out [N,3], converged [N] (may be NULL); queue_counter: device int32 [8], ZERO on entry:
 * [0] scratch (ray queue); statistics of the launch: [1] network evaluations, [2] rounds summed over the CTAs, [3] rounds that ran the
 * network, [4] rounds of the longest CTA. Bit-identical per ray to the masked Python loop on the per-op kernels. */
int psdf_sdf_sphere_trace(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                          const float* shift, const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob,
                          int nr_iters, float sdf_multiplier, float sdf_converged_tresh, const uint8_t* occupancy, int V, float extent,
                          const float trans[3], float sphere_radius, const float sphere_center[3], float* pos_out, uint8_t* converged,
                          int* queue_counter, void* stream);
/* psdf_sdf_sphere_trace at either input width and with either boundary primitive (sphere_trace with occupancy_grid and time_val,
 * sdf_utils.py:120-218). pos_dim 3, or 4: the network input is (x, y, z, time_val), time_val one fp32 per launch; positions, directions
 * and steps stay 3-D. boundary_kind 0: bounding sphere, boundary = {radius, centre x, y, z, -, -}; 1: box (AABB.check_point_inside_primitive,
 * aabb.py:28-43), boundary = {max bounds x, y, z, translation x, y, z}, a point is inside when min < p - t < max per coordinate with
 * min = -max. The occupancy grid, when given, replaces the boundary test as in psdf_sdf_sphere_trace. Other arguments as there;
 * psdf_sdf_sphere_trace is the (3, sphere) case. Returns PSDF_ERR_UNSUPPORTED for another pos_dim or boundary_kind. */
int psdf_sdf_sphere_trace_dim(int pos_dim, float time_val, int boundary_kind, const float boundary[6], int N, int L, int T, const float* pos,
                              const float* dirs, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                              float points_scaling, int hidden, int out_dim, const uint8_t* blob, int nr_iters, float sdf_multiplier,
                              float sdf_converged_tresh, const uint8_t* occupancy, int V, float extent, const float trans[3],
                              float* pos_out, uint8_t* converged, int* queue_counter, void* stream);
/* Training backward of psdf_sdf_fused_forward (double backward of encoding + MLP on the tensor cores, weight gradients formed on
 * chip; the lattice scatter is a second kernel at full occupancy):
 * upstream gradients g_sdf [N], g_grad [N,3], g_geom [N,out_dim-1] (any may be NULL) -> grad_lattice (+=), weight gradients
 * gW_l [N_l, K_l] (+=) and bias gradients gb_l [N_l] (+=). workspace: psdf_sdf_fused_backward_workspace_bytes(N) bytes of
 * scratch, per 128-sample tile 64 KB for the encoder operand tile (written and re-read by the same CTA) and 64 KB for the
 * per-level encoder gradients handed to the scatter kernel (16 bytes per sample and level, sized for 32 levels). Replaces
 * loss.backward() through SDF.get_sdf_and_gradient (models.py:199-259). */
long long psdf_sdf_fused_backward_workspace_bytes(int N);
int psdf_sdf_fused_backward(int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor, const float* shift,
                            const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, const float* g_sdf,
                            const float* g_grad, const float* g_geom, float* grad_lattice, uint8_t* workspace, float* gW0, float* gW1,
                            float* gW2, float* gW3, float* gb0, float* gb1, float* gb2, float* gb3, void* stream);
/* ---------------------------------------------------------------- fused colour network (RGB.forward, permuto_sdf_py/models/models.py:309-420)
 * encoding(points) | SH_5(dirs) | normalize(sdf_grad) | geom [N,32] -> 4-layer GELU MLP (in -> h1 -> h2 -> h3 -> 3) on the tensor
 * cores; out [N,3] is the linear output (colour calibration + sigmoid: psdf_calib_sigmoid_*). Weights are passed as a packed
 * operand blob (psdf_rgb_mlp_pack of the already Lipschitz-normalised matrices W_l [N_l,K_l] + biases); L % 4 == 0,
 * in_dim = 2L + 64 <= 128, h* <= 128 and % 16 == 0. */
long long psdf_rgb_mlp_blob_bytes(int in_dim, int h1, int h2, int h3, int out_dim);
int psdf_rgb_mlp_pack(int in_dim, int h1, int h2, int h3, int out_dim, const float* W0, const float* b0, const float* W1, const float* b1,
                      const float* W2, const float* b2, const float* W3, const float* b3, uint8_t* blob, void* stream);
int psdf_rgb_fused_forward(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                           const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                           int h1, int h2, int h3, const uint8_t* blob, float* out, void* stream);

/* backward of psdf_rgb_fused_forward: g_out [N,3] = d loss / d out -> grad_lattice (+=), g_sdf_grad [N,3] (=), g_geom [N,32] (=),
 * weight gradients gW_l [N_l,K_l] (+=, wrt the normalised matrices) and bias gradients gb_l (+=). workspace:
 * psdf_rgb_fused_backward_workspace_bytes(N) bytes of scratch. */
/* psdf_sdf_fused_backward over up to three independent sample sets in ONE launch (N_i = 0: unused set); every set has its own
 * positions and upstream gradients, the accumulated parameter gradients are shared. The sets share one last partial wave instead
 * of paying one each. */
long long psdf_sdf_fused_backward_multi_workspace_bytes(int N0, int N1, int N2);
int psdf_sdf_fused_backward_multi(int L, int T, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                                  float points_scaling, int hidden, int out_dim, const uint8_t* blob, int N0, const float* pos0,
                                  const float* g_sdf0, const float* g_grad0, const float* g_geom0, int N1, const float* pos1,
                                  const float* g_sdf1, const float* g_grad1, const float* g_geom1, int N2, const float* pos2,
                                  const float* g_sdf2, const float* g_grad2, const float* g_geom2, float* grad_lattice, uint8_t* workspace,
                                  float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1, float* gb2, float* gb3, void* stream);
/* ---------------------------------------------------------------- space-time SDF (SDF(in_channels=4, ...), train_4d_sdf.py:185)
 * The fused SDF pair at either input width, pos_dim first; pos_dim 3 is psdf_sdf_fused_forward / psdf_sdf_fused_backward_multi, pos_dim 4
 * takes space-time positions [N,4] (x, y, z, t) whose scale / shift rows have 4 columns. Both widths give 2L + 4 encoder columns (concat
 * column 2L + 3 holds t * points_scaling), so the blob of psdf_sdf_mlp_pack serves both. grad / g_grad are [N,3] for both: the SPATIAL
 * derivatives d sdf / d (x, y, z), which is all train_4d_sdf.py:212-217 reads of model.get_sdf_and_gradient (it keeps [:, 0:3] of the
 * [N,4] gradient); the time derivative is not formed. The backward's tangent direction is (g_grad, 0). The workspace does not depend on
 * pos_dim (psdf_sdf_fused_backward_multi_workspace_bytes). Any other pos_dim: PSDF_ERR_UNSUPPORTED. Replaces
 * model.get_sdf_and_gradient(points_time, iter_nr) (models.py:199-259) and loss.backward() through it (train_4d_sdf.py:212, 237). */
int psdf_sdf_fused_forward_dim(int pos_dim, int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor,
                               const float* shift, const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob,
                               float* sdf, float* grad, float* geom, void* stream);
int psdf_sdf_fused_backward_multi_dim(int pos_dim, int L, int T, const float* lattice, const float* scale_factor, const float* shift,
                                      const float* window, float points_scaling, int hidden, int out_dim, const uint8_t* blob, int N0,
                                      const float* pos0, const float* g_sdf0, const float* g_grad0, const float* g_geom0, int N1,
                                      const float* pos1, const float* g_sdf1, const float* g_grad1, const float* g_geom1, int N2,
                                      const float* pos2, const float* g_sdf2, const float* g_grad2, const float* g_geom2, float* grad_lattice,
                                      uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1, float* gb2,
                                      float* gb3, void* stream);
long long psdf_rgb_fused_backward_workspace_bytes(int N);
int psdf_rgb_fused_backward(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                            const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                            int h1, int h2, int h3, const uint8_t* blob, const float* g_out, float* grad_lattice, float* g_sdf_grad,
                            float* g_geom, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1,
                            float* gb2, float* gb3, void* stream);

/* ---------------------------------------------------------------- fused background network (NerfHash.forward, permuto_sdf_py/models/models.py:425-563)
 * encoding(pos [N,4]) (D = 4, concat points) -> trunk in -> 64 -> 64 -> 64 -> 65 (GELU between layers); density = softplus(z[:,0]);
 * [gelu(z[:,1:65]) | SH_4(dirs)] -> 64 -> 64 -> 3 (GELU between layers) = rgb_raw, before colour calibration and sigmoid. Seven layers on
 * the tensor cores; weights are passed as a packed operand blob (psdf_bg_mlp_pack of the seven torch.nn.Linear weights W_l [N_l,K_l] and
 * biases of mlp_feat_and_density and mlp_rgb). in_dim = 2L + 4, L % 4 == 0, pad16(in_dim) <= 64 (L <= 28). */
long long psdf_bg_mlp_blob_bytes(int in_dim);
int psdf_bg_mlp_pack(int in_dim, const float* W0, const float* b0, const float* W1, const float* b1, const float* W2, const float* b2,
                     const float* W3, const float* b3, const float* W4, const float* b4, const float* W5, const float* b5, const float* W6,
                     const float* b6, uint8_t* blob, void* stream);
int psdf_bg_fused_forward(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                          const float* shift, const float* window, float points_scaling, const uint8_t* blob, float* rgb_raw, float* density,
                          void* stream);
/* NerfHash.forward at either input width (permuto_sdf_py/models/models.py:425-563; train_nerf.py:164-165 builds NerfHash(3) for the
 * foreground and NerfHash(4) for the background): pos [N, pos_dim], pos_dim 3 or 4, otherwise the arguments of psdf_bg_fused_forward
 * (the scale / shift rows of the encoding have pos_dim columns). Both widths give 2L + 4 encoder columns, so the blob of psdf_bg_mlp_pack
 * serves both. psdf_bg_fused_forward is the pos_dim = 4 case. */
int psdf_nerf_fused_forward(int pos_dim, int N, int L, int T, const float* pos, const float* dirs, const float* lattice,
                            const float* scale_factor, const float* shift, const float* window, float points_scaling, const uint8_t* blob,
                            float* rgb_raw, float* density, void* stream);
/* NerfHash.get_only_density (permuto_sdf_py/models/models.py:528-550) of the foreground NerfHash(3): encoding(pos [N,3]) -> trunk ->
 * density [N] = softplus(z[:,0]), no colour head and no view directions. The blob of psdf_bg_mlp_pack (the head's blocks are not read);
 * the density equals psdf_nerf_fused_forward(3, ...)'s bit for bit. Row limits and PSDF_ERR_UNSUPPORTED cases of
 * psdf_nerf_fused_forward at pos_dim 3; N == 0 is a no-op; rows >= N are not written. */
int psdf_nerf_density_forward(int N, int L, int T, const float* pos, const float* lattice, const float* scale_factor, const float* shift,
                              const float* window, float points_scaling, const uint8_t* blob, float* density, void* stream);
/* backward of psdf_bg_fused_forward (loss.backward() through NerfHash.forward, first order): g_rgb_raw [N,3], g_density [N] ->
 * grad_lattice (+=), weight gradients gW_l [N_l,K_l] (+=) and bias gradients gb_l (+=). workspace:
 * psdf_bg_fused_backward_workspace_bytes(N) bytes of scratch. Launches the tensor-core kernel, then the lattice-scatter kernel. */
long long psdf_bg_fused_backward_workspace_bytes(int N);
int psdf_bg_fused_backward(int N, int L, int T, const float* pos, const float* dirs, const float* lattice, const float* scale_factor,
                           const float* shift, const float* window, float points_scaling, const uint8_t* blob, const float* g_rgb_raw,
                           const float* g_density, float* grad_lattice, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3,
                           float* gW4, float* gW5, float* gW6, float* gb0, float* gb1, float* gb2, float* gb3, float* gb4, float* gb5,
                           float* gb6, void* stream);
/* backward of psdf_nerf_fused_forward (loss.backward() through NerfHash.forward), arguments of psdf_bg_fused_backward after pos_dim;
 * workspace: psdf_bg_fused_backward_workspace_bytes(N). psdf_bg_fused_backward is the pos_dim = 4 case. */
int psdf_nerf_fused_backward(int pos_dim, int N, int L, int T, const float* pos, const float* dirs, const float* lattice,
                             const float* scale_factor, const float* shift, const float* window, float points_scaling, const uint8_t* blob,
                             const float* g_rgb_raw, const float* g_density, float* grad_lattice, uint8_t* workspace, float* gW0, float* gW1,
                             float* gW2, float* gW3, float* gW4, float* gW5, float* gW6, float* gb0, float* gb1, float* gb2, float* gb3,
                             float* gb4, float* gb5, float* gb6, void* stream);
/* background compositing with the colour head folded in (one thread per ray): Colorcal.calib_RGB_samples_packed + sigmoid of x_raw [N,3]
 * (models.py:677-741; img_idx [R] per ray, weight_delta / bias may be NULL: no calibration), then VolumeRenderingNerf.compute_weights +
 * integrate (volume_rendering_modules.py:61-89): alpha = 1 - exp(-density dt), T = exclusive cumprod(1 - alpha + 1e-7), w = alpha T,
 * bg_rgb [R,3] = sum w rgb. The backward takes g_bg_rgb [R,3] and writes g_x [N,3], g_density [N] (rows of the rays) and adds the
 * calibration gradients (may be NULL). */
int psdf_nerf_bg_composite_forward(PSDF_RSP, const float* x_raw, const float* density, const float* dt, const int* img_idx,
                                   const float* weight_delta, const float* bias, int fixed_img, float* bg_rgb, void* stream);
int psdf_nerf_bg_composite_backward(PSDF_RSP, const float* x_raw, const float* density, const float* dt, const int* img_idx,
                                    const float* weight_delta, const float* bias, int fixed_img, const float* g_bg_rgb, float* g_x,
                                    float* g_density, float* g_weight_delta, float* g_bias, void* stream);

/* foreground NeRF compositing and the loss of train_nerf.py (one thread per ray, samples left to right): colour head as in
 * psdf_nerf_bg_composite_forward, VolumeRenderingNerf.compute_weights + integrate (volume_rendering_modules.py:61-89),
 * bg_transmittance = the transmittance of the ray's last sample (VolumeRenderingGPU.cuh:400-416; 1 for a ray without samples),
 * pred_rgb = sum w rgb + bg_transmittance bg_rgb (train_nerf.py:76-95; bg_rgb [R,3] or NULL), weights_sum [R] = sum w, and
 * loss [1] = ((gt - pred)^2 hit).mean() + mask_weight BCE(weights_sum.clip(1e-3, 1 - 1e-3), gt_mask) (train_nerf.py:176-182; gt_mask [R]
 * or NULL: no mask term), terms [2] = {loss_rgb, BCE mean}. hit [R] u8. acc [3] scratch: zero before the first call, left zero by every
 * call. Deterministic mode: fixed-point sums. gt_rgb == NULL renders: no loss (hit, acc, loss, terms unused), and pred_rgb_bg [R,3]
 * (may be NULL) receives bg_transmittance bg_rgb.
 * The backward differentiates that loss (seed 1): g_x [N,3] and g_density [N] on the rows of the rays (=; other rows untouched),
 * g_bg_rgb [R,3] (=, with bg_rgb), calibration gradients (+=; may be NULL). torch's conventions: clamp passes the gradient on the closed
 * interval, BCE backward (x - y) / max(x (1 - x), 1e-12). */
int psdf_nerf_loss_forward(PSDF_RSP, const float* x_raw, const float* density, const float* dt, const int* img_idx, const float* weight_delta,
                           const float* bias, int fixed_img, const float* bg_rgb, const float* gt_rgb, const uint8_t* hit, const float* gt_mask,
                           float mask_weight, float* pred_rgb, float* weights_sum, float* bg_transmittance, float* pred_rgb_bg, float* acc,
                           float* loss, float* terms, void* stream);
int psdf_nerf_loss_backward(PSDF_RSP, const float* x_raw, const float* density, const float* dt, const int* img_idx, const float* weight_delta,
                            const float* bias, int fixed_img, const float* bg_rgb, const float* gt_rgb, const uint8_t* hit, const float* gt_mask,
                            float mask_weight, const float* pred_rgb, const float* weights_sum, const float* bg_transmittance, float* g_x,
                            float* g_density, float* g_bg_rgb, float* g_weight_delta, float* g_bias, void* stream);

/* ---------------------------------------------------------------- direct (autograd-free) training iteration
 * The reference's iteration (permuto_sdf_py/train_permuto_sdf.py:311-422) spends ~70 one-block PyTorch launches between its big kernels
 * (schedule ramps, Lipschitz normalisation, calibration, loss reductions, zero-fills, gradient adds). These entry points fold them into
 * the neighbouring kernels; permuto_sdf_b200/train.py Trainer._iteration_direct strings them together. */
/* two independent sample sets in one psdf_sdf_fused_forward launch (N1 = 0: unused); grad / geom may be NULL per set */
int psdf_sdf_fused_forward_multi(int L, int T, const float* lattice, const float* scale_factor, const float* shift, const float* window,
                                 float points_scaling, int hidden, int out_dim, const uint8_t* blob, int N0, const float* pos0, float* sdf0,
                                 float* grad0, float* geom0, int N1, const float* pos1, float* sdf1, float* grad1, float* geom1, void* stream);
/* psdf_sdf_mlp_pack + the end-of-iteration counters in the same launch: step_dev [1] (device int, AdamW step count) += 1 and
 * it_dev [1] (device float, iteration number) += 1; either may be NULL */
int psdf_sdf_mlp_pack_advance(int in_dim, int hidden, int out_dim, const float* W0, const float* b0, const float* W1, const float* b1,
                              const float* W2, const float* b2, const float* W3, const float* b3, uint8_t* blob, int* step_dev, float* it_dev,
                              void* stream);
/* psdf_rgb_fused_backward with g_sdf_grad accumulated (+=) instead of written */
int psdf_rgb_fused_backward_acc(int N, int L, int T, const float* pos, const float* dirs, const float* sdf_grad, const float* geom, int geom_dim,
                                const float* lattice, const float* scale_factor, const float* shift, const float* window, float points_scaling,
                                int h1, int h2, int h3, const uint8_t* blob, const float* g_out, float* grad_lattice, float* g_sdf_grad,
                                float* g_geom, uint8_t* workspace, float* gW0, float* gW1, float* gW2, float* gW3, float* gb0, float* gb1,
                                float* gb2, float* gb3, void* stream);
/* psdf_neus_render_loss_forward / _backward with the colour head (Colorcal.calib_RGB_samples_packed + sigmoid, models.py:395-414,677-741)
 * and the curvature term (models.py:283-294) folded in: x_raw [N,3] is the colour network's linear output; the backward returns
 * g_sdf [n_rows], g_grad [n_rows,3] (compositing + eikonal + curvature), g_x [n_rows,3], g_grad_shifted [n_rows,3] (curvature term wrt
 * the gradients at the shifted points; grad_shifted NULL: no curvature term), accumulates the calibration gradients (+=, may be NULL)
 * and zero-fills rows [nr_valid_dev[0], n_rows) (nr_valid_dev NULL: no tail). curv_scale weighs the curvature MEAN over
 * nr_samples_dev[0] (or max_nr_samples) rows; scale_eik is divided by the same count. */
int psdf_neus_head_loss_forward(PSDF_RSP, const float* sdf, const float* grad, const float* x_raw, const float* dirs, const float* dt,
                                const float* inv_s_dev, float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb,
                                const float* gt_mask, const uint8_t* hit, const int* img_idx, const float* weight_delta, const float* bias,
                                int fixed_img, float* alpha, float* transmittance, float* weights, float* pred_rgb, float* weights_sum,
                                float* bg_transmittance, float* ray_loss, void* stream);
int psdf_neus_head_loss_backward(PSDF_RSP, const float* sdf, const float* grad, const float* x_raw, const float* dirs, const float* dt,
                                 const float* inv_s_dev, float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb,
                                 const float* gt_mask, const uint8_t* hit, const int* img_idx, const float* weight_delta, const float* bias,
                                 int fixed_img, const float* alpha, const float* transmittance, const float* pred_rgb, const float* weights_sum,
                                 const float* bg_transmittance, float scale_rgb, float scale_mask, float scale_eik, const int* nr_samples_dev,
                                 const float* grad_shifted, float curv_scale, const float* curv_scale_dev, int n_rows, const int* nr_valid_dev,
                                 float* g_sdf, float* g_grad, float* g_x, float* g_grad_shifted, float* g_weight_delta, float* g_bias,
                                 void* stream);
/* the same pair for scenes without masks (train_permuto_sdf.py:149-163): bg_rgb [R,3] (psdf_nerf_bg_composite_forward) is blended in
 * behind every ray, as psdf_neus_render_loss_* do; the backward also writes g_bg_rgb [R,3]. */
int psdf_neus_head_bg_loss_forward(PSDF_RSP, const float* sdf, const float* grad, const float* x_raw, const float* dirs, const float* dt,
                                   const float* inv_s_dev, float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb,
                                   const float* gt_mask, const uint8_t* hit, const int* img_idx, const float* weight_delta, const float* bias,
                                   int fixed_img, const float* bg_rgb, float* alpha, float* transmittance, float* weights, float* pred_rgb,
                                   float* weights_sum, float* bg_transmittance, float* ray_loss, void* stream);
int psdf_neus_head_bg_loss_backward(PSDF_RSP, const float* sdf, const float* grad, const float* x_raw, const float* dirs, const float* dt,
                                    const float* inv_s_dev, float cos_anneal_ratio, const float* cos_anneal_dev, const float* gt_rgb,
                                    const float* gt_mask, const uint8_t* hit, const int* img_idx, const float* weight_delta, const float* bias,
                                    int fixed_img, const float* bg_rgb, const float* alpha, const float* transmittance, const float* pred_rgb,
                                    const float* weights_sum, const float* bg_transmittance, float scale_rgb, float scale_mask, float scale_eik,
                                    const int* nr_samples_dev, const float* grad_shifted, float curv_scale, const float* curv_scale_dev, int n_rows,
                                    const int* nr_valid_dev, float* g_sdf, float* g_grad, float* g_x, float* g_grad_shifted, float* g_bg_rgb,
                                    float* g_weight_delta, float* g_bias, void* stream);
/* Forward-only NeuS compositing of a rendered frame: VolumeRenderingNeus.compute_weights + integrate of the colour and of the SDF gradient
 * (permuto_sdf_py/volume_rendering/volume_rendering_modules.py:129-176) and the background blend of run_net
 * (permuto_sdf_py/train_permuto_sdf.py:133-162), with the colour head (calibration + sigmoid) folded in. It is the render mode of the kernel
 * behind psdf_neus_head_loss_forward: the same alpha / transmittance chain and colour head, no loss terms, nothing stored per sample.
 * sdf [N], grad [N,3] (d sdf / dx), x_raw [N,3] (colour network's linear output), dirs [N,3], dt [N], inv_s_dev [1] (device, clipped to
 * [1e-6,1e6] inside); img_idx [R] / weight_delta / bias [nr_imgs,3] may be NULL (no calibration); bg_rgb [R,3] or NULL. Per ray:
 *   pred_rgb [R,3] = sum w sigmoid(head(x_raw)) + T_last bg_rgb, pred_rgb_bg [R,3] = T_last bg_rgb (only with bg_rgb, else not written),
 *   pred_normals [R,3] = F.normalize(sum w grad) (eps 1e-12), weights_sum [R,1] = sum w.
 * Skipped rays (no sample, or end > max_nr_samples): pred_rgb = the background term, normal 0, weights_sum 0. */
int psdf_neus_render_forward(PSDF_RSP, const float* sdf, const float* grad, const float* x_raw, const float* dirs, const float* dt,
                             const float* inv_s_dev, float cos_anneal_ratio, const int* img_idx, const float* weight_delta, const float* bias,
                             int fixed_img, const float* bg_rgb, float* pred_rgb, float* pred_rgb_bg, float* pred_normals, float* weights_sum,
                             void* stream);
/* schedule ramps from the device-resident iteration (map_range_val, permuto_sdf_py/utils/common_utils.py:156-160): out[i] = out0 +
 * (out1 - out0) / (in1 - in0) * (clamp(it, in0, in1) - in0); kinds[i] = 1 / 2: exp(10 * ramp) unclipped / clipped to [1e-6, 1e6]
 * (inv_s of SingleVarianceNetwork with a forced variance). params [n,4] = {in0, in1, out0, out1} and kinds [n] are HOST arrays, n <= 8;
 * it_dev [1] device float or NULL (then it_host). */
int psdf_iter_scalars(int n, const float* params, const int* kinds, const float* it_dev, float it_host, float* out, void* stream);
/* psdf_lipschitz_normalize of the four colour-MLP matrices + psdf_rgb_mlp_pack of the result in one launch */
int psdf_lipschitz_pack4(int in_dim, int h1, int h2, int h3, int out_dim, const float* W0, const float* b0, const float* c0, const float* W1,
                         const float* b1, const float* c1, const float* W2, const float* b2, const float* c2, const float* W3, const float* b3,
                         const float* c3, uint8_t* blob, void* stream);
/* psdf_lipschitz_normalize_backward of the four layers in one launch: G_l = d loss / d W_eff_l is consumed and reset to zero,
 * grad_W_l (+=), grad_c_l (+=); lip_weight != 0 adds d (lip_weight * prod_l softplus(c_l)) / d c_l (LipshitzMLP.lipshitz_bound_full) */
int psdf_lipschitz_backward4(int in_dim, int h1, int h2, int h3, int out_dim, const float* W0, const float* c0, float* G0, float* gW0, float* gc0,
                             const float* W1, const float* c1, float* G1, float* gW1, float* gc1, const float* W2, const float* c2, float* G2,
                             float* gW2, float* gc2, const float* W3, const float* c3, float* G3, float* gW3, float* gc3, float lip_weight,
                             void* stream);
/* every scalar loss term of the iteration + the weighted total + the off-surface gradient seed in one launch (see csrc/iter_glue.cu);
 * acc [8] scratch: zero before the first call, left zero by every call; terms [12] = {sum L1, sum BCE, sum eikonal, mean curvature,
 * mean off-surface, Lipschitz bound, valid rows, divisor of the per-sample means, loss_rgb, loss_eikonal, unused, unused} */
int psdf_loss_terms(int N, const int* nr_valid_dev, const int* nr_mean_dev, const float* grad, const float* grad_shifted, int R,
                    const float* ray_loss, int n_off, const float* sdf_off, float* g_off, float c_rgb, float c_mask, float w_eik, float w_curv,
                    const float* w_curv_dev, float w_off, float w_lip, const float* lip_c0, const float* lip_c1, const float* lip_c2,
                    const float* lip_c3, float* acc, float* loss, float* terms, void* stream);
/* loss of one sphere-fit iteration (train_permuto_sdf.py:323-331, sdf_loss_sphere in permuto_sdf_utils.py:53-77) in one launch:
 *   loss = w_sdf mean((sdf - (|pos - center| - radius) s)^2) + w_eik mean((|grad| - s)^2),  s = distance_scale
 * pos [N,3], sdf [N], grad [N,3] (d sdf / d pos) -> g_sdf [N] = d loss / d sdf, g_grad [N,3] = d loss / d grad (=; zero where
 * |grad| = 0, as torch's norm backward), loss [1], terms [2] = {mean sdf term, mean eikonal term}. center[3] is a HOST array.
 * acc [4] scratch: zero before the first call, left zero by every call. Deterministic mode: fixed-point sums. */
int psdf_sphere_fit_loss(int N, const float* pos, const float* sdf, const float* grad, float radius, const float center[3], float distance_scale,
                         float w_sdf, float w_eik, float* g_sdf, float* g_grad, float* acc, float* loss, float* terms, void* stream);
/* points of one SDF-from-point-cloud iteration (train_sdf_from_mesh.py:119-123) in one launch (csrc/surface_fit.cu):
 *   x [Ns+No,3] = rows idx [Ns] (int64) of the cloud pts [P,3] (index_select), then the box rows u01 [No,3] * size - size / 2 +
 *   translation (AABB.rand_points_inside, permuto_sdf_py/utils/aabb.py:110-114, each operation rounded on its own as torch does);
 *   n [Ns,3] = rows idx of the normals nrm [P,3]. box_size / box_translation are HOST arrays. Ns = 0 is AABB.rand_points_inside from a
 *   given draw (pts, nrm, idx and n may then be NULL). An index outside [0, P) gives a NaN row. More than 2^31 - 1 floats in x or in the
 *   cloud: PSDF_ERR_UNSUPPORTED. */
int psdf_surface_fit_points(int P, int Ns, int No, const float* pts, const float* nrm, const long long* idx, const float* u01,
                            const float box_size[3], const float box_translation[3], float* x, float* n, void* stream);
/* points of one space-time iteration (train_4d_sdf.py:200-208): psdf_surface_fit_points with 4-column rows. x [Ns+No,4] = rows idx of the
 * cloud pts [P,4] (x, y, z, t), then the box rows u01 [No,3] * size - size / 2 + translation followed by the time draw ut [No,1]
 * (torch.cat([aabb.rand_points_inside(No), torch.rand(No, 1)], 1)); n [Ns,3] = rows idx of the normals nrm [P,3]. More than 2^31 - 1
 * floats in x or in the cloud: PSDF_ERR_UNSUPPORTED. */
int psdf_spacetime_fit_points(int P, int Ns, int No, const float* pts, const float* nrm, const long long* idx, const float* u01, const float* ut,
                              const float box_size[3], const float box_translation[3], float* x, float* n, void* stream);
/* sdf_loss (permuto_sdf_py/utils/sdf_utils.py:16-57, eik_clamp=None) times scale (train_sdf_from_mesh.py:135-136) in one launch over the
 * Ns surface rows followed by the No box rows of sdf [Ns+No], grad [Ns+No,3] (d sdf / d x), with the normals nrm [Ns,3]:
 *   loss = scale (w_eik mean_all |‖grad‖ - 1| + w_nrm mean_surf (1 - cos(grad, nrm)) + w_sdf mean_surf |sdf| + w_off mean_box exp(-100 |sdf|))
 * -> g_sdf [Ns+No] = d loss / d sdf, g_grad [Ns+No,3] = d loss / d grad (=, torch's autograd conventions: sign(0) = 0, a zero norm
 * backward at ‖grad‖ = 0, F.cosine_similarity with eps 1e-8), loss [1], terms [4] = the unweighted means {eikonal, normal, sdf, off}.
 * Ns >= 1 and No >= 1 (a mean over no rows is NaN in the reference). acc [5] scratch: zero before the first call, left zero by every
 * call. Deterministic mode: fixed-point sums. */
int psdf_surface_fit_loss(int Ns, int No, const float* sdf, const float* grad, const float* nrm, float w_eik, float w_nrm, float w_sdf,
                          float w_off, float scale, float* g_sdf, float* g_grad, float* acc, float* loss, float* terms, void* stream);
/* Sphere.rand_points_inside (src/Sphere.cu) from ONE uniform draw u01 [3,n]: rows = phi / (2 pi), (cos(theta) + 1) / 2, u */
int psdf_sphere_rand_points_inside_u01(int n, float radius, const float* u01, float* out, void* stream);

/* ---------------------------------------------------------------- marching cubes (csrc/marching_cubes.cu)
 * Replace skimage.measure.marching_cubes as extract_mesh_from_sdf_model calls it (permuto_sdf_py/utils/sdf_utils.py:280-283), on a volume
 * [N0, N1, N2] (axis 0 = x) streamed in slabs along axis 0. A slab is S >= 1 cell slices: vol points at S + 1 slices [N1, N2] starting at
 * global slice i0; last != 0 when its final slice is the volume's last. A corner is inside when value < threshold (NaN: outside). One vertex
 * per crossing grid edge, at the corner plus t = (threshold - f_lo) / (f_hi - f_lo) along the edge (fp32, each operation rounded), and
 * mapped to (x / div) * mul + off with affine_div_mul_off (a HOST array; {1, 1, 0} keeps index space). Vertices slice by slice (in-plane
 * axis-1 edges, in-plane axis-2 edges, each row-major in (j, k), then the axis-0 edges to the next slice), faces cell by cell in row-major
 * (i, j, k) order and in table order within a cell, so the output does not depend on the slab split. The triangle table is generated at
 * load: face segments that cut off the inside corners of ambiguous faces, closed loops oriented inside -> outside (right-hand normal),
 * fanned from their smallest edge (DESIGN.md §5a).
 * Per slab: psdf_marching_cubes_count -> counts [3] (device int64) = {vertices the slab emits, triangles, crossing edges including the
 * in-plane edges of its final slice}; the caller allocates verts [counts[0], 3] (float) and faces [counts[1], 3] (int32) and calls
 * psdf_marching_cubes_emit with the same slab, workspace and vertex_base = vertices emitted by earlier slabs; face entries are global vertex
 * ids, so vertex_base + counts[2] must stay below 2^31. The in-plane vertices of a slab's final slice are emitted by the next slab.
 * workspace: psdf_marching_cubes_workspace_bytes(S, N1, N2) bytes, PSDF_ERR_UNSUPPORTED for a slab whose edges or triangles could exceed
 * 2^31 - 1 (and for S < 1, N1 < 2 or N2 < 2). */
long long psdf_marching_cubes_workspace_bytes(int S, int N1, int N2);
int psdf_marching_cubes_count(int S, int N1, int N2, int i0, int last, float threshold, const float* vol, uint8_t* workspace, long long* counts,
                              void* stream);
int psdf_marching_cubes_emit(int S, int N1, int N2, int i0, int last, float threshold, const float* vol, long long vertex_base,
                             const float affine_div_mul_off[3], uint8_t* workspace, float* verts, int* faces, void* stream);

/* ---------------------------------------------------------------- mesh connected components (csrc/mesh_components.cu)
 * Connected components of the vertex graph of an indexed triangle mesh: V vertices, faces [F,3] int32, each face joining its three
 * vertices. The label of a vertex is the smallest vertex index of its component, so the labels depend only on the partition and the
 * vertex numbering: the same bits for any face order and on every run (lock-free union-find that links the larger root under the smaller,
 * integer atomics for every count). A vertex that no face references is a component of its own, with 0 faces.
 * workspace: psdf_mesh_components_workspace_bytes(V, F) = 256 + 8 V bytes; PSDF_ERR_UNSUPPORTED when V or F is 2^31 or more,
 * PSDF_ERR_ARG when negative. psdf_mesh_components fills it, and the caller may read it once the stream reaches that point:
 *   int64 info[4] at byte 0 = {number of components, faces with an index outside [0, V), largest key, 0},
 *   int32 labels [V] at byte 256, int32 face_counts [V] at byte 256 + 4 V (faces per component, indexed by label; each face counts
 *   for the component of its first vertex, entries of non-root vertices are 0).
 * The largest component is the one with the most faces, ties broken by the smallest label: largest key = (face count << 32) |
 * (2^32 - 1 - label), 0 for V = 0. A face with an index outside [0, V) is neither linked nor counted and nothing out of range is touched;
 * info[1] reports such faces, and the result is then not that of the mesh: callers check info[1] and refuse it. */
long long psdf_mesh_components_workspace_bytes(long long nr_vertices, long long nr_faces);
int psdf_mesh_components(int V, int F, const int* faces, uint8_t* workspace, void* stream);
/* keep [V] (uint8 / bool) from a workspace psdf_mesh_components filled for the same mesh: largest != 0 keeps the vertices of the largest
 * component (min_faces ignored), else those of components with at least min_faces faces (min_faces < 0: PSDF_ERR_ARG; 0 keeps every
 * vertex). */
int psdf_mesh_components_keep(int V, int largest, long long min_faces, const uint8_t* workspace, uint8_t* keep, void* stream);

/* ---------------------------------------------------------------- mesh decimation and vertex normals (csrc/mesh_decimate.cu)
 * Garland-Heckbert edge collapse in parallel rounds of independent collapses, on verts [V,3] (float) and faces [F,3] (int32), V and F
 * below 2^31. Built with -fmad=false: each fp64 / fp32 operation below is rounded as written, in the order written (oracle/decimate.py
 * restates it and matches bit for bit). Positions enter fp64 exactly (p = double(fp32)). The output is the same bits on every run; it
 * depends on the face order (edge ids are face corners).
 * CSR: the faces of each vertex. Faces with an index outside [0, V) or a repeated vertex are counted (info[0], info[1]) and left out.
 * Quadrics (begin): face t = (i0, i1, i2): N = (p1 - p0) x (p2 - p0), l = sqrt((Nx Nx + Ny Ny) + Nz Nz); l = 0 adds nothing; n = N / l,
 *   d = -((nx p0x + ny p0y) + nz p0z), w = l * 0.5, q = w * (x y) for the pairs {xx, xy, xz, xd, yy, yz, yd, zz, zd, dd} of (nx, ny, nz, d).
 *   Q[v] = sum of q over v's faces in ascending face order from 0. Collapsing b into a sets Q[a] = Q[a] + Q[b].
 * Locks (begin): half-edge (u, v) of a face (v the corner after u) locks u and v unless exactly one face of u holds u -> v and exactly one
 *   holds v -> u (boundary, an edge of three or more faces, inconsistent orientation).
 * Candidates: half-edge (u, v) at corner k of face f with u < v, id c = 3 f + k; it needs exactly one u -> v and one v -> u (face g) among
 *   u's faces, not both ends locked, and neither end in more than 64 faces (which bounds a candidate's work to 64^2 face reads). Survivor a = the locked end, else u; b = the other. Opposite vertices w (of f) != x (of g), each in
 *   more than 3 faces. Link: exactly 2 neighbours of b (the corners that follow b in its faces), other than a, lie in a face of a.
 * Position: Q = Q[a] + Q[b]. A locked a stays. Else with the cofactors c00 = Q4 Q7 - Q5 Q5, c01 = Q2 Q5 - Q1 Q7, c02 = Q1 Q5 - Q4 Q2,
 *   c11 = Q0 Q7 - Q2 Q2, c12 = Q1 Q2 - Q0 Q5, c22 = Q0 Q4 - Q1 Q1, det = (Q0 c00 + Q1 c01) + Q2 c02, tr = (Q0 + Q4) + Q7: when
 *   |det| > 1e-12 ((tr tr) tr), x = -(((c00 Q3 + c01 Q6) + c02 Q8) / det) and likewise with (c01, c11, c12) and (c02, c12, c22); x is taken,
 *   rounded to fp32, when |x - m|^2 <= |pb - pa|^2 with m = (pa + pb) * 0.5 (fp64, dot = (xx + yy) + zz). Otherwise the least error of
 *   pa, pb, then the fp32 midpoint (pa + pb) * 0.5f, a later one only when strictly smaller.
 * Error: r_i = ((Q row i . (x, y, z)) + Q row i's 4th entry) left to right, err = ((x r0 + y r1) + z r2) + r3, at double(fp32 position).
 * Validity: every face of a and of b except f and g keeps dot(N_before, N_after) > 0 (fp64, N as for the quadrics) with a or b moved.
 * Key = (fp32 bits of float(err > 0 ? err : 0)) << 33 | c, UINT64_MAX when any check fails. best[v] = min key of v's candidates,
 *   best2[v] = min best over v and the vertices of its faces; a candidate is chosen when its key == best2[u] == best2[v], so chosen
 *   collapses neither share nor neighbour a vertex. When more than `allowed` are chosen, those with the `allowed` smallest keys are applied.
 * Apply: position and Q to a, b -> a in b's faces, f and g dropped, removed[b] = 1, faces compacted in order; the caller's F shrinks by
 *   2 * applied.
 * Workspace: psdf_mesh_decimate_workspace_bytes(V, F) ~ 113 B per vertex + 37 B per face (sections each padded to 256 B):
 *   int64 info[8] at byte 0 = {faces with an index outside [0, V), faces that repeat a vertex, collapses chosen in the last round, collapses
 *   applied in it, threshold key, 0, 0, 0}, then int64 CSR offsets [V + 1], int32 counts [V], int32 CSR faces [3F], int64 scan tile sums,
 *   fp64 quadrics [V][10], uint64 best [V], best2 [V], uint8 locks [V], uint64 chosen keys [V / 2 + 1], uint64 keys [3F] + 8 B (the
 *   compaction's int64 prefix [F + 1] and int32 faces [3F] in the same bytes), uint8 dropped [F]. The normals' workspace
 *   (psdf_mesh_normals_workspace_bytes ~ 12 B per vertex + 12 B per face) is the first five sections.
 *   Both return PSDF_ERR_UNSUPPORTED when V or F is 2^31 or more and PSDF_ERR_ARG when negative.
 * psdf_mesh_decimate_begin: clears removed [V] (uint8), counts bad faces into info, builds the sorted CSR, the locks and the quadrics. Bad
 *   faces are left out, so nothing out of range is touched; the caller checks info[0] and info[1] and stops.
 * psdf_mesh_decimate_round: one round on the current faces [F] (F <= F0, the count given to begin, which sized the workspace); at most
 *   `allowed` collapses; verts, faces and removed are updated in place; info[2], info[3] tell what it did (info[3] = 0: no edge passes).
 * psdf_mesh_normals: normals [V,3] (float) = n / sqrtf((nx nx + ny ny) + nz nz) of n = the fp32 sum, in ascending face order from 0, of
 *   (p1 - p0) x (p2 - p0) (fp32, x = ay bz - az by) over v's faces; 0 when that length is 0. info[0] and info[1] count the bad faces as
 *   begin does (they are left out; the caller refuses them).
 * Cost: begin sorts each vertex's faces by heap sort (O(d log d) at valence d); twins are looked up in the list of the end with fewer
 *   faces; every other step reads each vertex's faces a bounded number of times, so a round is linear in the mesh. */
long long psdf_mesh_decimate_workspace_bytes(long long nr_vertices, long long nr_faces);
long long psdf_mesh_normals_workspace_bytes(long long nr_vertices, long long nr_faces);
int psdf_mesh_decimate_begin(int V, int F, const float* verts, const int* faces, uint8_t* workspace, uint8_t* removed, void* stream);
int psdf_mesh_decimate_round(int V, int F0, int F, long long allowed, float* verts, int* faces, uint8_t* workspace, uint8_t* removed,
                             void* stream);
int psdf_mesh_normals(int V, int F, const float* verts, const int* faces, uint8_t* workspace, float* normals, void* stream);

/* ---------------------------------------------------------------- mesh subdivision (csrc/mesh_subdivide.cu)
 * One round of midpoint (smooth = 0) or Loop (smooth != 0) subdivision of verts [V,3] (float) and faces [F,3] (int32): every face becomes
 * four. Built with -fmad=false: each fp32 operation below is rounded as written, in the order written (oracle/subdivide.py restates it and
 * matches bit for bit). The output depends only on V's bits and F, the same bits on every run.
 * Input: faces with an index outside [0, V) or a repeated vertex are counted (info[0], info[1]) and left out; the caller refuses them.
 *   Vertices without faces are carried over unchanged.
 * Edges: corner k of face f is the half-edge F[f][k] -> F[f][(k + 1) % 3], id 3 f + k. The faces of an undirected edge {u, v} are those
 *   that hold u and v; the edge is interior when there are exactly two, a crease otherwise (one, or three and more). Each edge gets one new
 *   vertex; they are numbered V + j in ascending order of the edge's smallest corner id, so the order depends on F alone.
 * Faces: face f = (v0, v1, v2) with edge vertices e01, e12, e20 (of its corners 0, 1, 2) becomes faces 4f .. 4f + 3 = (v0, e01, e20),
 *   (e01, v1, e12), (e20, e12, v2), (e01, e12, e20): the winding is kept, so a closed, oriented mesh stays closed and oriented.
 * Midpoint: edge vertex = 0.5f * (pu + pv); old vertices do not move.
 * Loop, edge vertices: interior edge of corner (u -> v) of face f with w the third vertex of f and x that of the other face:
 *   0.375f * (pu + pv) + 0.125f * (pw + px); crease edge: the midpoint. Sums of two points are commutative in fp32, so the order of u, v
 *   and of w, x does not matter.
 * Loop, old vertices: n = v's distinct neighbours, k = those joined to v by a crease edge.
 *   k = 0: beta = 0.1875f (n = 3), else 3.0f / float(8 n); w = 1.0f - float(n) * beta; p = w * pv + beta * s, where s = the fp32 sum of
 *     the neighbours' positions from 0.0f in ascending vertex index (s = s + pn).
 *   k = 2: p = 0.75f * pv + 0.125f * (pa + pb) with a < b the two crease neighbours.
 *   Otherwise (corners, non-manifold vertices) v does not move.
 *   beta is Warren's simplification, which libigl's loop uses as far as we recall; its source is not at hand, so this is unverified.
 *   Every product above is per coordinate: s * (x, y, z) = (s x, s y, s z).
 * Workspace: psdf_mesh_subdivide_workspace_bytes(V, F) ~ 12 B per vertex + 72 B per face (sections each padded to 256 B): int64 info[4]
 *   at byte 0 = {faces with an index outside [0, V), faces that repeat a vertex, edges E, 0}, then int64 CSR offsets [V + 1], int32 counts
 *   [V], int32 CSR faces [3F], int32 CSR neighbours [6F] (the two other corners of each of those faces), int64 scan tile sums, int32 edge
 *   owners [3F] (the smallest corner id of each corner's edge), int64 edge ids [3F + 1] (exclusive prefix of the corners that own their
 *   edge). PSDF_ERR_UNSUPPORTED when V or 4 F is 2^31 or more (the output faces are int32 rows), PSDF_ERR_ARG when negative.
 * psdf_mesh_subdivide_count: builds the CSR, counts bad faces into info[0], info[1] and the edges into info[2]. The caller reads info once,
 *   refuses bad faces, checks that V + E stays below 2^31 and allocates verts_out [V + E, 3] and faces_out [4F, 3].
 * psdf_mesh_subdivide_emit: with the workspace count filled for the same faces, writes verts_out and faces_out.
 * Cost: the Loop rule sorts each vertex's neighbour list by heap sort (O(d log d) at valence d); an edge's faces are looked up in the list
 *   of the end with fewer faces; every other step is one pass, so a round is linear in the mesh. */
long long psdf_mesh_subdivide_workspace_bytes(long long nr_vertices, long long nr_faces);
int psdf_mesh_subdivide_count(int V, int F, const int* faces, uint8_t* workspace, void* stream);
int psdf_mesh_subdivide_emit(int V, int F, int smooth, const float* verts, const int* faces, uint8_t* workspace, float* verts_out,
                             int* faces_out, void* stream);

/* ---------------------------------------------------------------- mesh ray casting (csrc/mesh_raycast.cu)
 * Any-hit queries of rays against the triangles of verts [V,3] (float) and faces [F,3] (int32) through a linear BVH, and per-vertex
 * ambient occlusion. Built with -fmad=false; oracle/raycast.py restates the triangle test and checks every answer by brute force.
 * Ray-triangle test (two-sided Moller-Trumbore, fp32, each operation rounded as written; dot(a, b) = (ax bx + ay by) + az bz, cross(a, b) =
 *   (ay bz - az by, az bx - ax bz, ax by - ay bx)): e1 = p1 - p0, e2 = p2 - p0, pv = cross(d, e2), det = dot(e1, pv); det == 0 or NaN
 *   misses. inv = 1.0f / det, tv = o - p0, u = dot(tv, pv) * inv, miss unless 0 <= u <= 1; qv = cross(tv, e1), v = dot(d, qv) * inv, miss
 *   unless v >= 0 and u + v <= 1; t = dot(e2, qv) * inv, hit iff tnear < t < tfar. A face that repeats a vertex has det == 0: never hit.
 * A ray is occluded exactly when some triangle passes the test; the tree only chooses which triangles are tested, so it changes no answer
 *   as long as its box test passes every box that holds a passing triangle:
 *   - Boxes are the exact fp32 min / max of their triangles' corners, grown at query time by pad = 2^-12 (s + max |o_k|), s the largest
 *     |coordinate| of the mesh. A passing (u, v, t) puts o + t d within |r| of the triangle, |r| <= c eps |tv| |d| |e1| |e2| / |det|
 *     (c ~ 10, eps = 2^-24, |tv| <= sqrt(3) (s + max |o_k|)); that is below pad unless the ray lies within about 1 degree of the triangle's
 *     plane (|det| < 2^-6 |d| |e1| |e2|). A ray that close to a far triangle's plane can pass the test by rounding alone, anywhere in that
 *     plane; such far passes are the one case where the answer can differ from the brute-force one. Zero-thickness boxes (axis-aligned
 *     triangles) are thickened by the pad, so origins on their planes lie inside.
 *   - Slab test: per axis, d_k == 0 requires lo_k - pad <= o_k <= hi_k + pad exactly (no 1/0, no 0 * inf); a d_k whose reciprocal is not
 *     finite leaves that axis out (conservative); otherwise the slab interval of (bound - o_k) * (1 / d_k). The box passes when
 *     max(tnear, slab starts) <= t1 + |t1| 2^-20 with t1 = min(tfar, slab ends): 2^-20 exceeds the 2 gamma_3 that covers the rounding of
 *     the slab arithmetic (Ize, Robust BVH ray traversal, 2013).
 *   - Traversal stack: 64 entries. Keys are the 30-bit Morton code of each centroid (within the centroids' bounds) with the sorted position
 *     breaking ties, so every internal node's common prefix length lies in [2, 63] and grows strictly from parent to child: at most 62
 *     internal nodes lie on a path, and only internal nodes are pushed, at most one per level.
 * Build: the faces are sorted by Morton code (four stable 8-bit radix passes), Karras' radix tree (2012) gives the F - 1 internal nodes
 *   (root 0), and the boxes are refit bottom-up. Faces with an index outside [0, V) are counted into info[0] (faces that repeat a vertex
 *   into info[1]; they are allowed) and get an empty box and NaN corners, so nothing out of range is read; the caller refuses them. F = 0
 *   (nothing is hit), F = 1, equal centroids and all faces at one point build a valid tree.
 * Workspace: psdf_mesh_bvh_workspace_bytes(V, F) ~ 152 B per face + 4 B per vertex (sections each padded to 256 B): int64 info[4] at byte
 *   0 = {faces with an index outside [0, V), faces that repeat a vertex, 0, 0}, uint32 bounds [8] (ordered keys of the centroid bounds, the
 *   bits of s), uint32 keys [2][F], int32 face ids [2][F], int32 radix histogram [256 ceil(F / 256)], int64 its prefix [+ 1], int64 scan
 *   tile sums, nodes [F - 1] of 64 B (both children's boxes, then the children; child >= F - 1 is leaf child - (F - 1)), int32 parents
 *   [2F - 1], int32 refit flags [F - 1], the sorted triangles [F] of 48 B (p0, p1, p2), int32 hit counts [V]. PSDF_ERR_UNSUPPORTED when V
 *   or F is 2^31 or more, PSDF_ERR_ARG when negative.
 * psdf_mesh_bvh_build: fills the workspace; queries pass the same V and F and read it.
 * psdf_mesh_occluded: hit_out[r] (uint8) = 1 when ray r (origins [R,3], dirs [R,3], any length) is occluded within (tnear, tfar); R is
 *   64-bit (PSDF_ERR_UNSUPPORTED above 256 (2^31 - 1)).
 * psdf_mesh_ambient_occlusion: V S rays, one per (vertex i, direction s), 64-bit ray ids: origin verts[i], direction dirs[s] [S,3], negated
 *   when dot(dirs[s], normals[i]) < 0 (fp32 as above), tnear = 1e-4f, tfar = +inf; vis_out[i] = float(S - hits) / float(S). Hits are
 *   integer counts, so the result is the same bits on every run.
 * Cost: build O(F) (sort, tree and refit are one pass each); a query visits the nodes whose padded boxes the ray meets. */
long long psdf_mesh_bvh_workspace_bytes(long long nr_vertices, long long nr_faces);
int psdf_mesh_bvh_build(int V, int F, const float* verts, const int* faces, uint8_t* workspace, void* stream);
int psdf_mesh_occluded(int V, int F, long long R, const float* origins, const float* dirs, float tnear, float tfar, const uint8_t* workspace,
                       uint8_t* hit_out, void* stream);
int psdf_mesh_ambient_occlusion(int V, int F, int S, const float* verts, const float* normals, const float* dirs, uint8_t* workspace,
                                float* vis_out, void* stream);

/* ---------------------------------------------------------------- image metrics (csrc/image_metrics.cu)
 * Per-image PSNR and SSIM of the reference's experiments/evaluation/evaluate_psnr.py, which scores each frame with piq.psnr and piq.ssim
 * (data_range = 1; kernel 11, sigma 1.5, k1 0.01, k2 0.03, downsampling on). x (the prediction) and y (the ground truth) are float images of
 * B x C x H x W values, each stored as [B,C,H,W] (nhwc = 0) or [B,H,W,C] (nhwc = 1); mask [B,H,W] or NULL. Offsets are 64-bit.
 * Before anything else, in this order:
 *   quantize_x != 0: x = min(255, max(0, rne(x * 255))) / 255 in fp32, create_my_images.py's 8-bit PNG round trip;
 *   mask: x = x m, y = y m (masked-out pixels stay in the means as exact matches, as in evaluate_psnr.py).
 * Everything after that is fp64:
 *   psdf_image_psnr: out[b] = -10 log10(mse + 1e-8), mse = the mean of (x - y)^2 over C, H, W at full resolution (piq.psnr);
 *   psdf_image_ssim: f = max(1, round(min(H, W) / 256)) (round half to even); f > 1 average-pools both images by f x f with stride f,
 *     dropping the remainder (F.avg_pool2d); H / f and W / f below 11: PSDF_ERR_ARG. Valid-mode sums with the normalised 11 x 11 Gaussian
 *     window give mu_x, mu_y, s_xx = W(x^2) - mu_x^2, s_yy, s_xy = W(xy) - mu_x mu_y; cs = (2 s_xy + c2) / (s_xx + s_yy + c2),
 *     ss = (2 mu_x mu_y + c1) / (mu_x^2 + mu_y^2 + c1) cs with c1 = 0.01^2, c2 = 0.03^2; out[b] = the mean of ss over C and the
 *     (H/f - 10)(W/f - 10) positions (piq.ssim's _ssim_per_channel, then the mean over channels).
 * out [B] (double). Partial sums go to the workspace, psdf_image_metrics_workspace_bytes(B, C, H, W) bytes (PSDF_ERR_ARG for a size below
 * 1, PSDF_ERR_UNSUPPORTED for B > 65535 or a size of 2^31 or more); their number depends only on the image size and they are added in a
 * fixed order, so a call gives the same bits on every run. Invalid arguments: PSDF_ERR_ARG before anything is launched. */
long long psdf_image_metrics_workspace_bytes(long long B, long long C, long long H, long long W);
int psdf_image_psnr(int B, int C, int H, int W, const float* x, int x_nhwc, const float* y, int y_nhwc, const float* mask, int quantize_x,
                    double* out, uint8_t* workspace, void* stream);
int psdf_image_ssim(int B, int C, int H, int W, const float* x, int x_nhwc, const float* y, int y_nhwc, const float* mask, int quantize_x,
                    double* out, uint8_t* workspace, void* stream);
/* psdf_adamw_step over up to 8 parameter groups in one launch: device-resident step count, per-group hyper_dev [2] = {lr, weight_decay};
 * gradients scaled by grad_scale and reset to zero. n_l % 4 == 0, 16-byte aligned pointers. n and the five tables of device addresses
 * (one entry per group) are HOST arrays. The step used is step_dev[0] + step_offset (step_offset = 1: the counter is advanced afterwards
 * by psdf_sdf_mlp_pack_advance). leave_room != 0: few resident blocks with more loads in flight each, so that kernels of another
 * stream (the next iteration's occupancy sampling) can be co-resident with the sweep. */
int psdf_adamw_multi_step(int n_groups, const long long* n, const uint64_t* param, const uint64_t* grad, const uint64_t* exp_avg,
                          const uint64_t* exp_avg_sq, const uint64_t* hyper_dev, float beta1, float beta2, float eps, const int* step_dev,
                          int step_offset, float grad_scale, int leave_room, void* stream);

/* ---------------------------------------------------------------- dense fused AdamW (torch.optim.AdamW / apex FusedAdam math,
 * train_permuto_sdf.py:293-304); step >= 1 is the incremented step count; grad is multiplied by grad_scale and, when
 * zero_grad != 0, reset to zero in the same pass. Pointers 16-byte aligned. step_dev [1] (device int32), when not NULL,
 * replaces `step` so that the call can be replayed from a CUDA graph; hyper_dev [2] (device float: lr, weight_decay), when not
 * NULL, replaces `lr` / `weight_decay` the same way (LR schedulers and the wd = 1.0 switch of train_permuto_sdf.py:400-403 edit
 * param_groups between replays of one captured graph). */
int psdf_adamw_step(long long n, float* param, float* grad, float* exp_avg, float* exp_avg_sq, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int step, const int* step_dev, const float* hyper_dev, float grad_scale, int zero_grad,
                    void* stream);

/* Data-parallel step without NCCL: gradient reduction + AdamW + parameter broadcast in ONE kernel over NVLink peer memory. This rank
 * owns the elements [shard_lo, shard_lo + n) of the group (both multiples of 4): it sums that shard of ALL ranks' gradient buffers
 * (peer loads), updates its local moments and writes the new parameters into ALL ranks' parameter buffers (peer stores).
 * grad_ptrs / param_ptrs: HOST arrays of `world` <= 8 device pointers (rank r's buffer of this group, peer-mapped here, e.g.
 * torch.distributed._symmetric_memory); mc_grad_ptr / mc_param_ptr: the NVSwitch MULTICAST mapping of the same two buffers (group base),
 * or 0: when given, the reduction is one multimem.ld_reduce (summed in the switch) and the broadcast one multimem.st per 16 bytes;
 * exp_avg / exp_avg_sq: local, full group size. world in {1, 2, 4, 8}. The caller puts a cross-rank barrier before
 * (gradients final) and after (parameters landed) the call and zeroes its own gradients afterwards. Replaces all-reduce + AdamW of
 * the reference's (non-existent) data-parallel loop: SURVEY.md 8(e). */
int psdf_adamw_dp_step(long long n, long long shard_lo, int world, int rank, const uint64_t* grad_ptrs, const uint64_t* param_ptrs,
                       uint64_t mc_grad_ptr, uint64_t mc_param_ptr, float* exp_avg, float* exp_avg_sq, float lr, float beta1, float beta2,
                       float eps, float weight_decay, int step, const int* step_dev, const float* hyper_dev, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif
