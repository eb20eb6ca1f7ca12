"""Hot-path drivers: sample creation, SDF importance resampling, the rendering forward (`run_net`), the
losses and one training iteration, and the sphere tracer.

Mirror of the orchestration in the reference (same function names and argument meaning):
  create_samples                   permuto_sdf_py/utils/nerf_utils.py:502-526
  importance_sampling_sdf_model    permuto_sdf_py/utils/sdf_utils.py:383-423
  sphere_trace                     permuto_sdf_py/utils/sdf_utils.py:120-218
  run_net / run_net_sphere_traced  permuto_sdf_py/train_permuto_sdf.py:111-170,211-242
  rgb_loss / eikonal_loss / ...    permuto_sdf_py/utils/permuto_sdf_utils.py:43-88
  train iteration                  permuto_sdf_py/train_permuto_sdf.py:311-422
"""
import math

import torch
import torch.nn.functional as F

from .graphs import capture, on_stream, run, sampler_graph_mode
from .models import RGB, SDF, Colorcal, DeviceIter, NerfHash, map_range_val
from .permuto_sdf import OccupancyGrid, PermutoSDF, RaySampler, RaySamplesPacked, Sphere, VolumeRendering


class HyperParams:
    """train_permuto_sdf.py:77-105 (defaults of the reference); the synthetic bench overrides sizes"""
    s_mult = 1.0
    lr = 1e-3
    nr_iter_sphere_fit = 4000
    forced_variance_finish_iter = 35000
    eikonal_weight = 0.04
    curvature_weight = 0.65
    lipshitz_weight = 3e-6
    mask_weight = 0.1
    offsurface_weight = 1e-4
    iter_start_reduce_curv = 50000
    iter_finish_reduce_curv = 50000 + 1001
    forced_variance_finish = 0.8
    use_occupancy_grid = True
    nr_samples_bg = 32
    min_dist_between_samples = 0.0001
    max_nr_samples_per_ray = 64
    nr_samples_imp_sampling = 16
    do_importance_sampling = True
    use_color_calibration = True
    nr_rays = 512
    sdf_geom_feat_size = 32
    sdf_nr_iters_for_c2f = 10000
    rgb_nr_iters_for_c2f = 1
    background_nr_iters_for_c2f = 1
    target_nr_of_samples = 512 * (64 + 16 + 16)
    with_mask = True
    # schedules of the reference loop (train_permuto_sdf.py:89-90,304,395-405,417-421)
    lr_milestones = (100000, 150000, 180000, 190000)
    lr_decay_gamma = 0.3
    lr_warmup_iters = 3000
    use_lr_schedule = True           # GradualWarmupScheduler(multiplier=1, total_epoch=3000) -> MultiStepLR(gamma=0.3)
    eikonal_weight_late = 0.01       # eikonal weight once iter >= iter_start_reduce_curv (:405)
    rgb_encoding_wd_late = 1.0       # weight decay of model_rgb_only_encoding from the same iteration on (:400-403)
    jitter_samples = None            # None: jitter while training (reference behaviour); True / False force it (tests)
    dp_world = 1                     # data-parallel ranks (set by Trainer.enable_data_parallel): sample-count weighting of the per-sample means
    adaptive_nr_rays = False         # nr_rays_to_create *= target_nr_of_samples / cur_nr_samples (:395-397); needs a host read per iteration
    nr_rays_bucket = 64              # adaptive ray counts are rounded to this multiple (bounded set of shapes / captured graphs)


def lr_schedule(hp, it):
    """learning rate used by optimizer.step() of (post-sphere-init) iteration `it` in the reference: the warm-up scheduler is
    created after the step of iteration 0 and stepped once per iteration (train_permuto_sdf.py:417-421), so iteration it >= 1
    runs with the value after `it` scheduler steps: base * it / 3000 up to 3000, then MultiStepLR counted from step 3001."""
    if not hp.use_lr_schedule or it <= 0:
        return hp.lr
    if it <= hp.lr_warmup_iters:
        return hp.lr * float(it) / hp.lr_warmup_iters
    epoch = it - (hp.lr_warmup_iters + 1)
    return hp.lr * hp.lr_decay_gamma ** sum(1 for m in hp.lr_milestones if epoch >= m)


def create_samples(with_mask, hyperparams, ray_origins, ray_dirs, jitter_samples, occupancy_grid, bounding_primitive):
    _, ray_t_entry, _, ray_t_exit, _ = bounding_primitive.ray_intersection(ray_origins, ray_dirs)
    if hyperparams.use_occupancy_grid and occupancy_grid is not None:
        fg = occupancy_grid.compute_samples_in_occupied_regions(ray_origins, ray_dirs, ray_t_entry, ray_t_exit,
                                                                hyperparams.min_dist_between_samples,
                                                                hyperparams.max_nr_samples_per_ray, jitter_samples)
    else:
        fg = RaySampler.compute_samples_fg(ray_origins, ray_dirs, ray_t_entry, ray_t_exit, hyperparams.min_dist_between_samples,
                                           hyperparams.max_nr_samples_per_ray, bounding_primitive.m_radius,
                                           bounding_primitive.m_center, jitter_samples)
    fg = fg.compact_to_valid_samples()
    bg = None
    if not with_mask:
        bg = RaySampler.compute_samples_bg(ray_origins, ray_dirs, ray_t_exit, hyperparams.nr_samples_bg, bounding_primitive.m_radius,
                                           bounding_primitive.m_center, jitter_samples, False)
    return fg, bg


# sphere_trace's loop as one tensor-core kernel instead of ~12 launches + a host sync per iteration (csrc/fused_sdf.cu k_sdf_sphere_trace:
# persistent CTAs over a global ray queue, finished slots refilled, resumable marches); no ray limit.
FUSED_SPHERE_TRACE = True
FUSED_SPHERE_TRACE_MAX_RAYS = 1 << 30
FUSED_IMPORTANCE_ROUND = True     # one launch per round (csrc/volrender.cu k_importance_round) instead of 9


def _imp_round(rsp, sdf, inv_s, inv_s_multiplier, ray_origins, ray_dirs, nr_imp, jitter):
    if FUSED_IMPORTANCE_ROUND:
        return VolumeRendering.importance_round(ray_origins, ray_dirs, rsp, sdf.contiguous(), inv_s, True, inv_s_multiplier, nr_imp, jitter)
    alpha = VolumeRendering.sdf2alpha(rsp, sdf, inv_s, True, inv_s_multiplier).clip(0.0, 1.0)
    T, _ = VolumeRendering.cumprod_alpha2transmittance(rsp, 1 - alpha + 1e-7)
    weights = alpha * T
    _, wsum_per_sample = VolumeRendering.sum_over_each_ray(rsp, weights)
    weights = weights / torch.clamp(wsum_per_sample, min=1e-6)
    cdf = VolumeRendering.compute_cdf(rsp, weights)
    return VolumeRendering.importance_sample(ray_origins, ray_dirs, rsp, cdf, nr_imp, jitter)


def importance_sampling_sdf_model(model_sdf, rsp, ray_origins, ray_dirs, ray_t_exit, iter_nr_for_anneal, nr_imp=16, jitter=None):
    inv_s_imp_sampling = 512
    jitter = model_sdf.training if jitter is None else bool(jitter)
    sdf, _ = model_sdf(rsp.samples_pos, iter_nr_for_anneal)
    rsp.set_sdf(sdf)
    imp = _imp_round(rsp, sdf, inv_s_imp_sampling, 1.0, ray_origins, ray_dirs, nr_imp, jitter)
    sdf_imp, _ = model_sdf(imp.samples_pos, iter_nr_for_anneal)
    imp.set_sdf(sdf_imp)
    rsp = VolumeRendering.combine_uniform_samples_with_imp(ray_origins, ray_dirs, ray_t_exit, rsp, imp).compact_to_valid_samples()
    # second round: sharper density, reuse the merged sdf (no network evaluation)
    imp = _imp_round(rsp, rsp.samples_sdf, inv_s_imp_sampling, 2.0, ray_origins, ray_dirs, nr_imp, jitter)
    rsp.remove_sdf()
    rsp = VolumeRendering.combine_uniform_samples_with_imp(ray_origins, ray_dirs, ray_t_exit, rsp, imp).compact_to_valid_samples()
    return rsp


def run_net_samples(with_mask, hyperparams, ray_origins, ray_dirs, model_sdf, occupancy_grid, iter_nr_for_anneal):
    """the sampling of run_net (train_permuto_sdf.py:111-135): occupancy-grid (or bounding-sphere) samples, compacted, then SDF
    importance resampling; background samples for scenes without masks. Jitters while model_sdf is training unless
    hyperparams.jitter_samples says otherwise. Call without autograd. -> (fg, bg or None)"""
    _, _, _, ray_t_exit, _ = model_sdf.boundary_primitive.ray_intersection(ray_origins, ray_dirs)
    jitter = model_sdf.training if getattr(hyperparams, "jitter_samples", None) is None else bool(hyperparams.jitter_samples)
    fg, bg = create_samples(with_mask, hyperparams, ray_origins, ray_dirs, jitter, occupancy_grid, model_sdf.boundary_primitive)
    if hyperparams.do_importance_sampling and fg.samples_pos.shape[0] != 0:
        fg = importance_sampling_sdf_model(model_sdf, fg, ray_origins, ray_dirs, ray_t_exit, iter_nr_for_anneal,
                                           hyperparams.nr_samples_imp_sampling, jitter=jitter)
    return fg, bg


def run_net(with_mask, hyperparams, ray_origins, ray_dirs, img_indices, model_sdf, model_rgb, model_bg, model_colorcal, occupancy_grid,
            iter_nr_for_anneal, cos_anneal_ratio, forced_variance, fused_loss=None):
    """train_permuto_sdf.py:88-177. With `fused_loss` (dict: gt_rgb, gt_mask, hit, w_eik, w_mask) the NeuS compositing and the
    rgb / mask / eikonal losses run in the fused kernel pair (csrc/neus_fused.cu); the result lands in fused_loss['loss']."""
    with torch.no_grad():
        fg, bg = run_net_samples(with_mask, hyperparams, ray_origins, ray_dirs, model_sdf, occupancy_grid, iter_nr_for_anneal)
        if getattr(hyperparams, "dp_world", 1) > 1:
            # per-sample means (eikonal, curvature) are means over the samples of all ranks: one 4-byte all-reduce of the count
            import torch.distributed as dist
            n_sum = fg.cur_nr_samples.to(torch.int32).clone()
            dist.all_reduce(n_sum, op=dist.ReduceOp.SUM)
            W = int(hyperparams.dp_world)
            fg.dp_mean_nr_samples = torch.div(n_sum + W // 2, W, rounding_mode="floor").to(torch.int32).clamp(min=1)
    if fg.samples_pos.shape[0] == 0:
        pred_rgb = torch.zeros_like(ray_origins)
        pred_normals = torch.zeros_like(ray_origins)
        sdf_gradients = torch.zeros_like(ray_origins)
        weights_sum = torch.zeros_like(ray_origins)[:, 0:1]
        bg_transmittance = torch.ones_like(ray_origins)[:, 0:1]
    elif fused_loss is not None:
        sdf, sdf_gradients, geom_feat = model_sdf.get_sdf_and_gradient(fg.samples_pos, iter_nr_for_anneal)
        rgb_samples = model_rgb(fg.samples_pos, fg.samples_dirs, sdf_gradients, geom_feat, iter_nr_for_anneal, model_colorcal, img_indices,
                                fg.ray_start_end_idx)
        vr = model_rgb.volume_renderer_neus
        inv_s = vr.deviation_network(forced_variance)
        vr.last_inv_s = inv_s.detach().clip(1e-6, 1e6)
        bg_rgb = None
        if not with_mask and bg is not None and bg.samples_pos_4d.shape[0] != 0:
            rgb_bg, density_bg = model_bg(bg.samples_pos_4d, bg.samples_dirs, iter_nr_for_anneal, model_colorcal, img_indices,
                                          ray_start_end_idx=bg.ray_start_end_idx)
            weights_bg, _, _ = model_bg.volume_renderer_nerf.compute_weights(bg, density_bg.view(-1, 1))
            bg_rgb = model_bg.volume_renderer_nerf.integrate(bg, rgb_bg, weights_bg)
        from .fused import neus_render_loss
        loss, pred_rgb, weights_sum, _, terms = neus_render_loss(fg, sdf, sdf_gradients, rgb_samples, inv_s, cos_anneal_ratio,
                                                                 fused_loss["gt_rgb"], fused_loss["gt_mask"], fused_loss["hit"],
                                                                 fused_loss["w_eik"], fused_loss["w_mask"], bg_rgb=bg_rgb)
        fused_loss["loss"], fused_loss["terms"] = loss, terms
        return pred_rgb, None, None, sdf_gradients, weights_sum, fg
    else:
        sdf, sdf_gradients, geom_feat = model_sdf.get_sdf_and_gradient(fg.samples_pos, iter_nr_for_anneal)
        rgb_samples = model_rgb(fg.samples_pos, fg.samples_dirs, sdf_gradients, geom_feat, iter_nr_for_anneal, model_colorcal, img_indices,
                                fg.ray_start_end_idx)
        weights, weights_sum, bg_transmittance, inv_s = model_rgb.volume_renderer_neus.compute_weights(fg, sdf, sdf_gradients,
                                                                                                       cos_anneal_ratio, forced_variance)
        pred_rgb = model_rgb.volume_renderer_neus.integrate(fg, rgb_samples, weights)
        pred_normals = F.normalize(model_rgb.volume_renderer_neus.integrate(fg, sdf_gradients, weights), dim=1)
    pred_rgb_bg = None
    if not with_mask and bg is not None and bg.samples_pos_4d.shape[0] != 0:
        rgb_bg, density_bg = model_bg(bg.samples_pos_4d, bg.samples_dirs, iter_nr_for_anneal, model_colorcal, img_indices,
                                      ray_start_end_idx=bg.ray_start_end_idx)
        weights_bg, _, _ = model_bg.volume_renderer_nerf.compute_weights(bg, density_bg.view(-1, 1))
        pred_rgb_bg = bg_transmittance.view(-1, 1) * model_bg.volume_renderer_nerf.integrate(bg, rgb_bg, weights_bg)
        pred_rgb = pred_rgb + pred_rgb_bg
    return pred_rgb, pred_rgb_bg, pred_normals, sdf_gradients, weights_sum, fg


def rgb_loss(gt_rgb, pred_rgb, does_ray_intersect_primitive):
    return ((gt_rgb - pred_rgb).abs() * does_ray_intersect_primitive * 1.0).mean()


def eikonal_loss(sdf_gradients):
    return ((torch.linalg.norm(sdf_gradients.reshape(-1, 3), ord=2, dim=-1) - 1.0) ** 2).mean()


def sdf_loss_sphere(points, sdf, sdf_gradients, sphere_radius, sphere_center, distance_scale=1.0):
    """permuto_sdf_utils.py sphere-init loss: |sdf - (||x-c|| - r)| + eikonal"""
    c = torch.as_tensor(sphere_center, dtype=points.dtype, device=points.device).view(1, 3)
    gt = ((points - c).norm(dim=-1, keepdim=True) - sphere_radius) * distance_scale
    loss_sdf = ((sdf - gt) ** 2).mean()
    loss_eik = ((sdf_gradients.norm(dim=-1) - distance_scale) ** 2).mean()
    return loss_sdf * 3e3 + loss_eik * 5e1, loss_sdf, loss_eik


def loss_sphere_init(nr_points, aabb, model, iter_nr_for_anneal, points=None, sphere_radius=0.3, sphere_center=(0, 0, 0)):
    """points: [nr_points, 3] to evaluate instead of a fresh aabb.rand_points_inside draw"""
    pts = aabb.rand_points_inside(nr_points=nr_points) if points is None else points
    sdf, grads, _ = model.get_sdf_and_gradient(pts, iter_nr_for_anneal)
    return sdf_loss_sphere(pts, sdf, grads, sphere_radius=sphere_radius, sphere_center=list(sphere_center))


def sphere_trace(nr_sphere_traces, ray_origins, ray_dirs, model, return_gradients, sdf_multiplier, sdf_converged_tresh,
                 occupancy_grid=None, time_val=None):
    """sdf_utils.py:120-218 (boolean-mask gather/scatter loop, as in the reference). model.boundary_primitive is a Sphere or an AABB.
    time_val: a space-time SDF (SDF(4, ...)) is traced at that time, as train_4d_sdf.py:268 does: the network sees (x, y, z, time_val),
    the traced points stay 3-D and the returned gradient is the spatial one ([:, 0:3] of the reference's [N,4] gradient)."""
    ray_points_entry, ray_t_entry, _, ray_t_exit, _ = model.boundary_primitive.ray_intersection(ray_origins, ray_dirs)
    has_occupancy = occupancy_grid is not None
    if has_occupancy:
        rsp = occupancy_grid.compute_first_sample_start_of_occupied_regions(ray_origins, ray_dirs, ray_t_entry, ray_t_exit)
        rsp = rsp.compact_to_valid_samples()
        pos, dirs = rsp.samples_pos, rsp.samples_dirs
        pos = pos + dirs * (1.0 / occupancy_grid.get_nr_voxels_per_dim()) * 0.5
    else:
        rsp = RaySamplesPacked(ray_origins.shape[0], ray_origins.shape[0])
        rsp.initialize_with_one_sample_per_ray(ray_points_entry, ray_dirs)
        pos, dirs = rsp.samples_pos, rsp.samples_dirs
    pts = pos.clone()
    converged = torch.zeros_like(pos)[:, 0:1].bool()

    def with_time(p):                   # the reference's torch.cat([p, torch.empty(n, 1).fill_(time_val)], 1)
        return p if time_val is None else torch.cat([p, torch.full((p.shape[0], 1), float(time_val), device=p.device)], 1)

    fused_tracer = FUSED_SPHERE_TRACE and getattr(model, "fused", None) is not None and 0 < pos.shape[0] <= FUSED_SPHERE_TRACE_MAX_RAYS
    if fused_tracer:
        # the whole loop below in one kernel (csrc/fused_sdf.cu k_sdf_sphere_trace): same per-ray arithmetic, no gather / scatter / sync
        pts, _ = model.fused.sphere_trace(pos, dirs, model.last_iter_nr, nr_sphere_traces, sdf_multiplier, sdf_converged_tresh,
                                          occupancy_grid if has_occupancy else None, time_val)
    for _ in range(0 if fused_tracer else nr_sphere_traces):
        sel = torch.logical_not(converged).view(-1)
        pos_u, dirs_u = pts[sel].contiguous(), dirs[sel].contiguous()
        if pos_u.shape[0] == 0:
            break
        sdf, _ = model(with_time(pos_u), model.last_iter_nr)
        pos_u = (pos_u + dirs_u * sdf * sdf_multiplier).contiguous()
        newly = (sdf.abs() < sdf_converged_tresh).view(-1)
        if has_occupancy:
            pos_u, within = occupancy_grid.advance_sample_to_next_occupied_voxel(dirs_u, pos_u)
        else:
            within = model.boundary_primitive.check_point_inside_primitive(pos_u)
        conv_u = torch.logical_or(newly, torch.logical_not(within.view(-1)))
        converged[sel] = torch.logical_or(converged[sel].view(-1), conv_u).view(-1, 1)
        pts[sel] = pos_u
    pts_t = with_time(pts).contiguous()
    if return_gradients and getattr(model, "fused", None) is not None:
        sdf, grads, geom = model.fused(pts_t, model.last_iter_nr, with_gradient=True)      # forward-mode normal, one kernel
    elif return_gradients:
        with torch.enable_grad():
            sdf, grads, geom = model.get_sdf_and_gradient(pts_t.detach().clone(), model.last_iter_nr)
            grads = grads.detach()[:, 0:3]
    else:
        sdf, geom = model(pts_t, model.last_iter_nr)
        grads = None
    rsp.samples_pos = pts
    return pts, sdf, grads, geom, rsp


def filter_unconverged_points(points, sdf, sdf_gradients, sdf_converged_tresh=0.01):
    """sdf_utils.py:221-231, as written there: rows whose SIGNED sdf is below the threshold count as converged (a point far inside the
    surface passes too) -> (points * c, sdf_gradients * c or None, c [N,1] float)"""
    is_sdf_converged = (sdf < sdf_converged_tresh) * 1.0
    points_converged = points * is_sdf_converged
    sdf_gradients_converged = sdf_gradients * is_sdf_converged if sdf_gradients is not None else None
    return points_converged, sdf_gradients_converged, is_sdf_converged


def run_net_sphere_traced(ray_origins, ray_dirs, hyperparams, model_sdf, model_rgb, occupancy_grid, iter_nr_for_anneal, nr_sphere_traces,
                          sdf_multiplier, sdf_converged_tresh):
    """train_permuto_sdf.py:211-242 without the frame->rays and image reshapes"""
    ray_end, _, ray_end_gradient, geom_feat_end, traced = sphere_trace(nr_sphere_traces, ray_origins, ray_dirs, model_sdf, True,
                                                                      sdf_multiplier, sdf_converged_tresh, occupancy_grid)
    within = model_sdf.boundary_primitive.check_point_inside_primitive(ray_end).view(-1)
    if hyperparams.use_occupancy_grid and occupancy_grid is not None:
        within = torch.logical_and(occupancy_grid.check_occupancy(ray_end).view(-1), within)
    weights = within.float().view(-1, 1).contiguous()
    vr = model_rgb.volume_renderer_neus
    pred_normals = F.normalize(vr.integrate(traced, ray_end_gradient.contiguous(), weights), dim=1)
    rgb_samples = model_rgb(traced.samples_pos, traced.samples_dirs, ray_end_gradient, geom_feat_end, iter_nr_for_anneal)
    pred_rgb = vr.integrate(traced, rgb_samples.contiguous(), weights)
    pred_weights_sum, _ = VolumeRendering.sum_over_each_ray(traced, weights)
    return pred_rgb, pred_normals, pred_weights_sum


def load_from_checkpoint(ckpt_path_full, model_sdf, model_rgb, model_bg, occupancy_grid, model_colorcal=None):
    """permuto_sdf_utils.py:222-237: <ckpt_path_full>/{sdf_model,rgb_model,nerf_hash_model_bg}.pt + grid_values.pt /
    grid_occupancy.pt, the files train_permuto_sdf.py:444-453 writes (same key names, so reference checkpoints load here and
    ours load there). Models that are None (no background network with --with_mask) are skipped."""
    import os
    dev = next(model_sdf.parameters()).device
    ld = lambda name: torch.load(os.path.join(ckpt_path_full, name), map_location=dev)
    model_sdf.load_state_dict(ld("sdf_model.pt"))
    model_rgb.load_state_dict(ld("rgb_model.pt"))
    if model_bg is not None and os.path.exists(os.path.join(ckpt_path_full, "nerf_hash_model_bg.pt")):
        model_bg.load_state_dict(ld("nerf_hash_model_bg.pt"))
    if model_colorcal is not None and os.path.exists(os.path.join(ckpt_path_full, "colorcal_model.pt")):
        model_colorcal.load_state_dict(ld("colorcal_model.pt"))
    for m in (model_sdf, model_rgb, model_bg):
        if m is not None:
            m.eval()
    if occupancy_grid is not None and os.path.exists(os.path.join(ckpt_path_full, "grid_values.pt")):
        occupancy_grid.set_grid_values(ld("grid_values.pt"))
        occupancy_grid.set_grid_occupancy(ld("grid_occupancy.pt"))


def run_net_in_chunks(ray_origins_full, ray_dirs_full, chunk_size, with_mask, hyperparams, model_sdf, model_rgb, model_bg, occupancy_grid,
                      iter_nr_for_anneal, cos_anneal_ratio, forced_variance):
    """train_permuto_sdf.py:172-209 without the frame -> rays / image reshapes: volume-render a full image chunk by chunk.
    -> (pred_rgb [R,3], pred_rgb_bg [R,3] or None, pred_normals [R,3], pred_weights_sum [R,1])"""
    nr_chunks = max(1, math.ceil(ray_origins_full.shape[0] / chunk_size))
    rgb_l, bg_l, nrm_l, ws_l = [], [], [], []
    with torch.no_grad():
        for o, d in zip(torch.chunk(ray_origins_full, nr_chunks), torch.chunk(ray_dirs_full, nr_chunks)):
            pred_rgb, pred_rgb_bg, pred_normals, _, weights_sum, _ = run_net(with_mask, hyperparams, o.contiguous(), d.contiguous(), None,
                                                                             model_sdf, model_rgb, model_bg, None, occupancy_grid,
                                                                             iter_nr_for_anneal, cos_anneal_ratio, forced_variance)
            rgb_l.append(pred_rgb.detach()); nrm_l.append(pred_normals.detach()); ws_l.append(weights_sum.detach())
            if pred_rgb_bg is not None:
                bg_l.append(pred_rgb_bg.detach())
    return torch.cat(rgb_l, 0), (torch.cat(bg_l, 0) if bg_l else None), torch.cat(nrm_l, 0), torch.cat(ws_l, 0)


class HostLoss:
    """Loss of an iteration on its way to the host: the 4-byte device -> pinned-host copy is queued right behind the iteration's
    forward/backward graph (BEFORE its optimizer step), float() / item() wait for that copy only. The host can therefore read the
    loss of iteration i and launch iteration i+1 while the optimizer step of iteration i is still running (Trainer.step_from_reel
    with loss_to_host=True). Valid until the next step of the same Trainer."""

    def __init__(self, host, event, dev):
        self.host, self.event, self.dev = host, event, dev

    def __float__(self):
        self.event.synchronize()
        return float(self.host[0])

    def item(self):
        return float(self)

    def detach(self):
        return self.dev


class Trainer:
    """State of one PermutoSDF training run on synthetic data (models, occupancy grid, optimizer) and its two phases:
      * the sphere-fit phase (train_permuto_sdf.py:323-331), `fit_sphere()`: hp.nr_iter_sphere_fit iterations that fit the SDF to a
        sphere of radius 0.3 before training; counted by `sphere_fit_iter`;
      * the per-iteration training step of train_permuto_sdf.py:311-422 after the fit, `step()`, with `--with_mask` semantics; counted
        by `iter_nr`, which the fit leaves at 0."""

    def __init__(self, hyperparams=None, nr_levels=24, capacity=2 ** 18, sdf_hidden=32, nr_images=8, occupancy_resolution=256,
                 seed=0, with_colorcal=True, optimizer="adamw", fused_inference=True, fused_training=True, fused_render=True, direct=None,
                 deterministic=False, fused_background=False):
        """direct: None = run the iteration through the autograd-free sequence of iteration.DirectIteration whenever the configuration
        allows it (fused kernels, flat-buffer optimizer, --with_mask); True = require it (raise otherwise); False = autograd formulation.
        deterministic: switch the library's deterministic mode on for this device (psdf_set_deterministic: order-independent gradient
        reductions, so runs with the same inputs give the same bits; the direct iteration is fully covered) -- or off (the default,
        float atomics).
        fused_background: run the background NerfHash of scenes without masks on the fused tensor-core kernels (csrc/fused_bg.cu)
        instead of the per-op encoding kernels + autograd; a background shape the kernels do not cover raises."""
        torch.manual_seed(seed)
        self.fused_render = fused_render
        self._fused_inference = fused_inference
        self.hp = hyperparams or HyperParams()
        self.aabb = Sphere(0.5, [0, 0, 0])
        hp = self.hp
        self.model_sdf = SDF(3, self.aabb, hp.sdf_geom_feat_size, hp.sdf_nr_iters_for_c2f, nr_levels, capacity, sdf_hidden).to("cuda")
        self.model_rgb = RGB(3, self.aabb, hp.sdf_geom_feat_size, hp.rgb_nr_iters_for_c2f, nr_levels, capacity).to("cuda")
        self.model_bg = None if hp.with_mask else NerfHash(4, self.aabb, hp.background_nr_iters_for_c2f, nr_levels, capacity).to("cuda")
        self.model_colorcal = Colorcal(nr_images, 0) if (hp.use_color_calibration and with_colorcal) else None
        self.occupancy_grid = OccupancyGrid(occupancy_resolution, 1.0, [0, 0, 0]) if hp.use_occupancy_grid else None
        from ._lib import call as _call
        _call("psdf_set_deterministic", 1 if deterministic else 0, nr_levels * capacity * 2, occupancy_resolution ** 3)
        # No silent fall-back: asking for the fused (tensor-core) path with a shape it does not cover raises here (FusedSDF / FusedRGB
        # say which constraint failed); the per-op path is only taken when the caller asks for it (fused_inference=False /
        # fused_training=False). `self.execution` records which path each model runs on.
        self.execution = {"sdf_inference": "per-op kernels", "sdf_training": "per-op kernels + autograd", "rgb": "per-op kernels + autograd",
                          "background": "per-op kernels + autograd" if self.model_bg is not None else None}
        if fused_inference:
            self.model_sdf.enable_fused_inference()
            self.execution["sdf_inference"] = "fused wgmma"
            if fused_training:
                self.model_sdf.enable_fused_training()
                self.model_rgb.enable_fused()
                self.execution["sdf_training"] = self.execution["rgb"] = "fused wgmma"
        if fused_background and self.model_bg is not None:
            self.model_bg.enable_fused()
            self.execution["background"] = "fused wgmma"
        groups = [{"params": list(self.model_sdf.parameters()), "weight_decay": 0.0, "lr": hp.lr, "name": "model_sdf"}]
        if self.model_bg is not None:
            groups.append({"params": list(self.model_bg.parameters()), "weight_decay": 0.0, "lr": hp.lr, "name": "model_bg"})
        groups.append({"params": self.model_rgb.parameters_only_encoding(), "weight_decay": 0.0, "lr": hp.lr, "name": "model_rgb_only_encoding"})
        groups.append({"params": self.model_rgb.parameters_all_without_encoding(), "weight_decay": 0.0, "lr": hp.lr,
                       "name": "model_rgb_all_without_encoding"})
        if self.model_colorcal is not None:
            groups.append({"params": list(self.model_colorcal.parameters()), "weight_decay": 1e-1, "lr": hp.lr, "name": "model_colorcal"})
        self.params = [p for g in groups for p in g["params"]]
        if optimizer == "fused":
            from .optim import FusedAdamW      # our dense AdamW kernel over flat buffers (csrc/optim.cu)
            self.optimizer = FusedAdamW(groups, betas=(0.9, 0.99), eps=1e-15, lr=hp.lr)
            for m in (self.model_sdf, self.model_rgb, self.model_bg):     # .grad buffers exist for good: scatter into them directly
                if m is not None:
                    m.encoding.grad_in_place = True
        else:
            self.optimizer = torch.optim.AdamW(groups, amsgrad=False, betas=(0.9, 0.99), eps=1e-15, weight_decay=0.0, lr=hp.lr)
        # the iteration itself: explicit kernel sequence (iteration.py) or torch.autograd around the same kernels
        from .iteration import DirectIteration
        self.fixed_random = None        # tests: {"offsurface_u01": [3,1024], "curvature_dirs": [N,3]} replace the torch RNG draws
        self._direct = None
        why = DirectIteration.unsupported_reason(self) if direct is not False else "disabled by the caller (direct=False)"
        if why is None:
            self._direct = DirectIteration(self)
        elif direct:
            raise RuntimeError("Trainer(direct=True): " + why)
        self.execution["iteration"] = "direct kernel sequence (iteration.py)" if self._direct is not None else "torch.autograd (%s)" % why
        self._direct_why = why
        self.execution["sphere_fit"] = None      # set by fit_sphere()
        self.iter_nr = 0
        self.sphere_fit_iter = 0        # sphere-fit iterations run so far (fit_sphere)
        self._fit = None                # device counters and graph slot (graphs.run) of the direct sphere fit
        self._cg = None                 # CUDA-graph state (enable_cuda_graph)
        self._dp = None                 # data-parallel state (enable_data_parallel)
        self._render = None             # workspaces of render()
        self.nr_rays_to_create = hp.nr_rays
        self.last = {}

    def save(self, ckpt_folder, experiment_name, iter_nr=None, with_optimizer=True):
        """train_permuto_sdf.py:444-453: every model's state_dict + the occupancy grid under <ckpt>/<experiment>/<iter>/models/;
        additionally (not in the reference) the optimizer moments and iteration number, so that a run resumes bit for bit"""
        import os
        it = self.iter_nr if iter_nr is None else iter_nr
        path = self.model_sdf.save(ckpt_folder, experiment_name, it)
        self.model_rgb.save(ckpt_folder, experiment_name, it)
        if self.model_bg is not None:
            self.model_bg.save(ckpt_folder, experiment_name, it, additional_name="_bg")
        if self.model_colorcal is not None:
            self.model_colorcal.save(ckpt_folder, experiment_name, it)
        if self.occupancy_grid is not None:
            torch.save(self.occupancy_grid.get_grid_values(), os.path.join(path, "grid_values.pt"))
            torch.save(self.occupancy_grid.get_grid_occupancy(), os.path.join(path, "grid_occupancy.pt"))
        if with_optimizer:
            torch.save(self._trainer_state(), os.path.join(path, "trainer_state.pt"))
        return path

    def _trainer_state(self):
        return {"optimizer": self.optimizer.state_dict(), "iter_nr": self.iter_nr, "nr_rays_to_create": self.nr_rays_to_create,
                "sphere_fit_iter": self.sphere_fit_iter}

    def _restore_trainer_state(self, sd):
        """inverse of _trainer_state(); sd None: no trainer_state.pt (a reference checkpoint). A state without `sphere_fit_iter` (older
        files, reference checkpoints) comes from a run past its sphere fit: the fit counts as finished."""
        if sd is not None:
            self.optimizer.load_state_dict(sd["optimizer"])
            self.iter_nr = int(sd["iter_nr"])
            self.nr_rays_to_create = int(sd.get("nr_rays_to_create", self.nr_rays_to_create))
        self.sphere_fit_iter = int(sd["sphere_fit_iter"]) if (sd is not None and "sphere_fit_iter" in sd) else int(self.hp.nr_iter_sphere_fit)

    def load(self, ckpt_path_full, with_optimizer=True):
        """inverse of save(); also reads checkpoints written by the reference (no trainer_state.pt: models + grid only).
        Parameters are copied into the existing storages, so the flat-buffer optimizer's views stay valid."""
        import os
        load_from_checkpoint(ckpt_path_full, self.model_sdf, self.model_rgb, self.model_bg, self.occupancy_grid, self.model_colorcal)
        st = os.path.join(ckpt_path_full, "trainer_state.pt")
        if with_optimizer and os.path.exists(st):
            self._restore_trainer_state(torch.load(st, map_location=next(self.model_sdf.parameters()).device))
        else:
            self._restore_trainer_state(None)
        if getattr(self.model_sdf, "fused", None) is not None:
            self.model_sdf.fused.repack()           # load_state_dict copies in place
        if self._cg is not None:
            self._cg["it_host"] = None              # device-resident iteration number is refreshed on the next step

    def set_analytic_scene(self, object_radius=0.3, inv_s=512.0):
        """occupancy of the analytic sphere SDF ||x|| - r through update_with_sdf (SURVEY.md 8d, C2)"""
        g = self.occupancy_grid
        pts = g.compute_grid_points(False)
        sdf = (pts.norm(dim=1, keepdim=True) - object_radius).contiguous()
        g.update_with_sdf(sdf, inv_s, 1e10, 1e-4)

    def draw(self, name, fn):
        """random draw `name` of the iteration: fn() (torch RNG) unless a test pinned it in self.fixed_random"""
        fr = self.fixed_random
        return fr[name] if (fr is not None and name in fr) else fn()

    def forward_backward(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, iter_nr_for_anneal, pre=None):
        """losses + backward of one iteration; parameter gradients are ACCUMULATED into .grad (the caller has run
        optimizer.zero_grad(); outside any graph capture). -> detached loss. pre: DirectIteration.sample_uniform() of these rays when
        it already ran as its own graph"""
        if self._direct is not None:
            loss = self._direct.run(ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, iter_nr_for_anneal, pre=pre)
            if loss is not None:
                return loss
        loss = self.losses(ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, iter_nr_for_anneal)
        loss.backward()
        return loss.detach()

    def losses(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, iter_nr_for_anneal):
        hp = self.hp
        cos_anneal_ratio = map_range_val(iter_nr_for_anneal, 0.0, hp.forced_variance_finish_iter, 0.0, 1.0)
        forced_variance = map_range_val(iter_nr_for_anneal, 0.0, hp.forced_variance_finish_iter, 0.3, hp.forced_variance_finish)
        with torch.no_grad():
            _, _, _, _, does_hit = self.aabb.ray_intersection(ray_origins, ray_dirs)
        fl = None
        if self.fused_render:
            fl = dict(gt_rgb=gt_rgb, gt_mask=gt_mask if hp.with_mask else None, hit=does_hit, w_eik=hp.eikonal_weight, w_mask=hp.mask_weight,
                      loss=None)
        pred_rgb, _, _, sdf_gradients, weights_sum, fg = run_net(hp.with_mask, hp, ray_origins, ray_dirs, img_indices, self.model_sdf,
                                                                 self.model_rgb, self.model_bg, self.model_colorcal, self.occupancy_grid,
                                                                 iter_nr_for_anneal, cos_anneal_ratio, forced_variance, fused_loss=fl)
        fused_done = fl is not None and fl["loss"] is not None
        if fused_done:
            loss = fl["loss"]      # rgb L1 + eikonal + mask terms, already weighted
            nr = fg.cur_nr_samples.clamp(min=1).float().squeeze(0) if RaySamplesPacked.static_capacity else max(fg.samples_pos.shape[0], 1)
            loss_rgb, loss_eik = fl["terms"][0] / (3.0 * ray_origins.shape[0]), fl["terms"][2] / nr
        else:
            loss_rgb = rgb_loss(gt_rgb, pred_rgb, does_hit)
            loss = loss_rgb
            loss_eik = eikonal_loss(sdf_gradients)
            loss = loss + loss_eik * hp.eikonal_weight
        gw_curv = map_range_val(iter_nr_for_anneal, hp.iter_start_reduce_curv, hp.iter_finish_reduce_curv, 1.0, 0.0)
        loss_curv = torch.zeros((), device=loss.device)
        if iter_nr_for_anneal < hp.iter_finish_reduce_curv and fg.samples_pos.shape[0] != 0:      # <=> gw_curv > 0
            if self.fused_render:
                rnd = self.draw("curvature_dirs", lambda: torch.randn_like(fg.samples_pos))
                loss_curv = self.model_sdf.curvature_loss(fg.samples_pos, sdf_gradients, iter_nr_for_anneal,
                                                          fg.cur_nr_samples if RaySamplesPacked.static_capacity else None, rnd=rnd)
                if getattr(fg, "dp_mean_nr_samples", None) is not None:       # mean over the samples of all ranks (see run_net)
                    loss_curv = loss_curv * (fg.cur_nr_samples.float() / fg.dp_mean_nr_samples.float()).squeeze(0)
            else:
                _, curv = self.model_sdf.get_sdf_and_curvature_1d_precomputed_gradient_normal_based(fg.samples_pos, sdf_gradients,
                                                                                                    iter_nr_for_anneal)
                if RaySamplesPacked.static_capacity:     # rows past the device-side sample count are padding
                    n_dev = fg.cur_nr_samples
                    valid = (torch.arange(curv.shape[0], device=curv.device, dtype=torch.int32) < n_dev).view(-1, 1)
                    loss_curv = torch.where(valid, curv, torch.zeros_like(curv)).sum() / n_dev.clamp(min=1).float().squeeze(0)
                else:
                    loss_curv = curv.mean()
            loss = loss + loss_curv * hp.curvature_weight * gw_curv
        if hp.use_occupancy_grid:
            u01 = self.draw("offsurface_u01", lambda: torch.rand(3, 1024, device=loss.device))
            off = self.aabb.rand_points_inside_u01(u01)
            sdf_rand, _ = self.model_sdf(off, iter_nr_for_anneal)
            loss = loss + torch.exp(-1e2 * torch.abs(sdf_rand)).mean() * hp.offsurface_weight
        if iter_nr_for_anneal >= hp.iter_start_reduce_curv:      # the bound is only part of the loss from here on
            loss_lip = self.model_rgb.mlp.lipshitz_bound_full()
            loss = loss + loss_lip.mean() * hp.lipshitz_weight
        if hp.with_mask and not fused_done:
            loss = loss + F.binary_cross_entropy(weights_sum.clip(1e-3, 1.0 - 1e-3), gt_mask) * hp.mask_weight
        self.last = dict(loss_rgb=loss_rgb.detach(), loss_eikonal=loss_eik.detach(), loss_curvature=loss_curv.detach(),
                         nr_samples=fg.samples_pos.shape[0], nr_samples_dev=fg.cur_nr_samples, fg=fg)
        return loss

    # ------------------------------------------------------------------------------------ data parallel (SURVEY.md 8e)
    def enable_data_parallel(self, world, overlap=False, mode="peer"):
        """Rays are sharded by rank, parameters replicated (same seed), gradients summed over the ranks and the mean folded into AdamW.
        The flat gradient buffer is reduced in buckets that overlap with compute instead of one blocking all-reduce between backward
        and optimizer:
          * the colour hash table's gradient (half of the bytes) is final as soon as the colour network's backward kernel has run --
            it runs FIRST in loss.backward() -- so its all-reduce is started right there and travels over NVLink while the SDF
            backward kernels run;
          * the rest is reduced after the backward while AdamW already sweeps the (reduced) colour hash table.
        Per-sample means (eikonal, curvature) are weighted by the sample counts of all ranks (run_net), so the averaged gradient is the
        gradient of the global batch. Works eagerly and inside the captured graphs (NCCL collectives are capturable)."""
        import torch.distributed as dist
        if not hasattr(self.optimizer, "flat_grad"):
            raise RuntimeError("data-parallel mode needs the flat-buffer optimizer (optimizer='fused')")
        self.hp.dp_world = int(world)
        if mode == "peer":
            # no all-reduce at all: one fused reduce + AdamW + broadcast kernel per parameter group over NVLink peer memory
            # (optim.FusedAdamW.enable_peer_step, csrc/optim.cu k_adamw_dp); the step runs eagerly behind the replayed iteration graph
            self.optimizer.enable_peer_step()
            self._dp = dict(world=int(world), mode="peer", work=None, dist=dist)
            if getattr(self.model_sdf, "fused", None) is not None:
                self.model_sdf.fused.repack()
            if self._cg is not None:
                self._cg["fb"], self._cg["opt"] = None, {}      # captured graphs point at the old buffers
            return
        gi = next(i for i, g in enumerate(self.optimizer.param_groups) if g.get("name") == "model_rgb_only_encoding")
        g = self.optimizer.param_groups[gi]
        self._dp = dict(world=int(world), mode="nccl", rgb_group=gi, off=g["_off"], n=g["_n"], overlap=bool(overlap), work=None, dist=dist)
        if overlap and getattr(self.model_rgb, "fused", None) is not None:
            self.model_rgb.fused.after_backward = self._dp_start_rgb_table_reduce
        if self._cg is not None:
            self._cg["fb"], self._cg["opt"] = None, {}      # graphs captured without the collectives are stale

    def _dp_start_rgb_table_reduce(self):
        dp = self._dp
        fg = self.optimizer.flat_grad
        dp["work"] = dp["dist"].all_reduce(fg[dp["off"]:dp["off"] + dp["n"]], op=dp["dist"].ReduceOp.SUM, async_op=True)

    def _dp_join_backward(self):
        """end of the backward: the early bucket's collective rejoins the stream (needed before a graph capture ends); if the colour
        network did not start it (modular path), nothing is pending"""
        dp = getattr(self, "_dp", None)
        if dp is not None and dp["work"] is not None:
            dp["work"].wait()
            dp["work"] = None
            dp["rgb_reduced"] = True

    def dp_reduce_gradients(self):
        """finish the data-parallel reduction WITHOUT stepping (tests / inspection): flat_grad <- mean over the ranks"""
        dp = self._dp
        dist, fg = dp["dist"], self.optimizer.flat_grad
        if dp["mode"] == "peer":
            dist.all_reduce(fg, op=dist.ReduceOp.SUM)
            fg.mul_(1.0 / dp["world"])
            return
        lo, hi = dp["off"], dp["off"] + dp["n"]
        if dp.pop("rgb_reduced", False):
            if lo > 0:
                dist.all_reduce(fg[:lo], op=dist.ReduceOp.SUM)
            if hi < fg.numel():
                dist.all_reduce(fg[hi:], op=dist.ReduceOp.SUM)
        else:
            dist.all_reduce(fg, op=dist.ReduceOp.SUM)
        fg.mul_(1.0 / dp["world"])

    def _dp_optimizer_step(self, rgb_reduced):
        """all-reduce of what is not reduced yet, overlapped with AdamW on the colour hash table; mean folded into the step"""
        dp = self._dp
        dist, fg, opt = dp["dist"], self.optimizer.flat_grad, self.optimizer
        scale = 1.0 / dp["world"]
        if dp["mode"] == "peer":
            opt.step(grad_scale=scale)
            return
        lo, hi = dp["off"], dp["off"] + dp["n"]
        if rgb_reduced:
            works = []
            if lo > 0:
                works.append(dist.all_reduce(fg[:lo], op=dist.ReduceOp.SUM, async_op=True))
            if hi < fg.numel():
                works.append(dist.all_reduce(fg[hi:], op=dist.ReduceOp.SUM, async_op=True))
            opt.step(grad_scale=scale, groups=[dp["rgb_group"]])
            for w in works:
                w.wait()
            opt.step(grad_scale=scale, groups=[i for i in range(len(opt.param_groups)) if i != dp["rgb_group"]], advance=False)
        else:
            dist.all_reduce(fg, op=dist.ReduceOp.SUM)
            opt.step(grad_scale=scale)

    def apply_schedules(self, it):
        """host-side schedule edits of one iteration, run between the loss and the optimizer step like the reference does
        (train_permuto_sdf.py:395-405,417-421): LR warm-up / decay, weight decay 1.0 on the colour hash table and eikonal weight
        0.01 once iter >= iter_start_reduce_curv (the new eikonal weight is seen by the NEXT iteration's loss, as in the reference,
        where the edit follows the loss computation). In CUDA-graph mode lr / weight decay reach the kernel through
        FusedAdamW.hyper_dev and the eikonal weight is part of the forward/backward graph's cache key."""
        hp = self.hp
        lr = lr_schedule(hp, it)
        late = it >= hp.iter_start_reduce_curv
        for g in self.optimizer.param_groups:
            g["lr"] = lr
            if late and g.get("name") == "model_rgb_only_encoding":
                g["weight_decay"] = hp.rgb_encoding_wd_late
        if late:
            hp.eikonal_weight = hp.eikonal_weight_late

    def adapt_nr_rays(self, cur_nr_samples):
        """train_permuto_sdf.py:395-397; the count is bucketed so that CUDA-graph mode sees a bounded set of ray counts"""
        hp = self.hp
        if not hp.adaptive_nr_rays or cur_nr_samples <= 0:
            return self.nr_rays_to_create
        n = int(self.nr_rays_to_create * float(hp.target_nr_of_samples) / cur_nr_samples)
        b = max(int(hp.nr_rays_bucket), 1)
        self.nr_rays_to_create = max(b, (n + b // 2) // b * b)
        return self.nr_rays_to_create

    def update_occupancy(self, iter_nr_for_anneal):
        """train_permuto_sdf.py:386-391 (every 8th iteration)"""
        with torch.no_grad():
            pts, idx = self.occupancy_grid.compute_random_sample_of_grid_points(256 * 256 * 4, True)
            sdf_grid, _ = self.model_sdf(pts, iter_nr_for_anneal)
            self.occupancy_grid.update_with_sdf_random_sample(idx, sdf_grid.contiguous(), self.model_rgb.volume_renderer_neus.get_last_inv_s(), 1e-4)

    def render(self, ray_origins, ray_dirs, chunk_size=None, iter_nr_for_anneal=None, cos_anneal_ratio=1.0, forced_variance=None):
        """Volume-render rays chunk by chunk on the fused kernels (render.VolumeRender): what run_net_in_chunks(ray_origins, ray_dirs,
        chunk_size, hp.with_mask, hp, model_sdf, model_rgb, model_bg, occupancy_grid, iter_nr_for_anneal, cos_anneal_ratio,
        forced_variance) computes, from the same samples. chunk_size: rays per chunk (default render.DEFAULT_CHUNK, at most
        render.VolumeRender.max_chunk(hp)); iter_nr_for_anneal: default self.iter_nr; forced_variance None: the learned variance.
        Samples are jittered while model_sdf is in training mode, as in run_net: put the models in eval() to render a frame.
        Reads no parameter gradient and changes no parameter, .grad, occupancy grid or iteration counter; without jitter it advances no
        generator. Raises when a model is not on the fused kernels.
        -> (pred_rgb [R,3], pred_rgb_bg [R,3] or None (scenes with masks), pred_normals [R,3], pred_weights_sum [R,1])"""
        from .render import DEFAULT_CHUNK, VolumeRender
        if self._render is None:
            self._render = VolumeRender(self)
        return self._render.render(ray_origins, ray_dirs, DEFAULT_CHUNK if chunk_size is None else chunk_size,
                                   self.iter_nr if iter_nr_for_anneal is None else iter_nr_for_anneal, cos_anneal_ratio, forced_variance)

    def _frame_models(self):
        return (self.model_sdf, self.model_rgb, self.model_bg, self.model_colorcal)

    def _frame_render(self, chunk_size):
        """render() with the settings of create_my_images.py: iteration 9999999, cos_anneal_ratio 1, hp.forced_variance_finish"""
        from .metrics import FRAME_ITER
        return lambda o, d: self.render(o, d, chunk_size, FRAME_ITER, 1.0, self.hp.forced_variance_finish)

    def render_frame(self, tensor_reel, img_idx, chunk_size=None):
        """Every pixel of image img_idx of a TensorReel, rendered as create_my_images.py renders a frame: the rays of
        PermutoSDF.rays_from_reel_indices, the models in eval mode (train flags restored afterwards), iteration 9999999, cos_anneal_ratio 1,
        hp.forced_variance_finish. Changes no parameter, .grad, occupancy grid, iteration counter or generator; raises as render() does.
        -> (rgb [1,3,H,W], unit normals in camera coordinates [1,3,H,W], weights sum [1,1,H,W]), channels-last views of the rendered rows.
        The normals are F.normalize(R n) with R the rotation of tf_cam_world = tf_world_cam^-1, so a zero normal stays zero."""
        from . import metrics
        (rgb, _, normals, wsum), H, W = metrics.render_frame("Trainer.render_frame", tensor_reel, img_idx, self._frame_models(),
                                                             self._frame_render(chunk_size))
        tf = tensor_reel.tf_world_cam_reel[int(img_idx)]
        R = torch.linalg.inv(tf.cpu())[0:3, 0:3].to(normals.device)
        normals = F.normalize(torch.matmul(R, normals.t()).t(), dim=1)
        return metrics.image(rgb, H, W), metrics.image(normals, H, W), metrics.image(wsum, H, W)

    def evaluate(self, tensor_reel, image_indices=None, chunk_size=None, quantize=True):
        """PSNR and SSIM of rendered frames, as create_my_images.py renders them (render_frame) and evaluate_psnr.py scores them: the
        colour 8-bit quantized when `quantize` (the PNG round trip), prediction and the reel's rgb multiplied by the reel's mask when it
        has one, then metrics.psnr and metrics.ssim. image_indices None: every image of the reel.
        -> {"image_indices", "psnr", "ssim" (fp64 per image, on the host), "psnr_mean", "ssim_mean"}"""
        from .metrics import evaluate_frames
        render = self._frame_render(chunk_size)
        return evaluate_frames("Trainer.evaluate", tensor_reel, image_indices, quantize, self._frame_models(), lambda o, d: render(o, d)[0])

    def step(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, update_occupancy=None, optimizer_step=True):
        """forward + losses + backward (+ optimizer). Returns the detached loss tensor (no host sync)."""
        self.model_sdf.train(); self.model_rgb.train()
        if self._cg is not None:
            return self._step_graphed(ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, update_occupancy, optimizer_step)
        it = self.iter_nr
        self.optimizer.zero_grad(set_to_none=False)
        loss = self.forward_backward(ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, it)
        self._dp_join_backward()
        if update_occupancy is None:
            update_occupancy = (it % 8 == 0)
        if update_occupancy and self.hp.use_occupancy_grid:
            self.update_occupancy(it)
        if self.hp.adaptive_nr_rays:
            self.adapt_nr_rays(int(self.last["nr_samples"]))
        self.apply_schedules(it)
        if optimizer_step:
            self.optimizer_step()
        self.iter_nr += 1
        return loss

    # ------------------------------------------------------------------------------------ sphere-fit phase
    def fit_sphere(self, nr_iters=None, nr_points=30000, radius=0.3, center=(0, 0, 0)):
        """The sphere-fit phase that precedes training (train_permuto_sdf.py:323-331): per iteration `nr_points` uniform points inside
        the bounding sphere, loss sdf_loss_sphere (3e3 mean (sdf - (|p - c| - r))^2 + 5e1 mean (|d sdf/dx| - 1)^2) and AdamW at the
        constant hp.lr over the SDF parameters only. The other groups' parameters and Adam moments do not change; FusedAdamW's single
        step count advances (apex FusedAdam advances every group's step, the reference's optimizer when apex is installed), torch AdamW
        creates no state for them. The fit iteration is the anneal iteration of the SDF coarse-to-fine window.
        Runs the rest of the phase, at most `nr_iters` iterations: min(nr_iters, hp.nr_iter_sphere_fit - sphere_fit_iter); iter_nr
        does not change. Whenever the trainer runs the direct iteration the fit is the direct kernel sequence (DirectIteration.sphere_fit),
        replayed from one captured graph after enable_cuda_graph(); otherwise loss_sphere_init + loss.backward().
        -> detached 0-d loss of the last iteration (no host sync), None when no iteration ran."""
        if self._dp is not None:
            raise RuntimeError("fit_sphere: the sphere fit runs on one GPU (the reference has no data-parallel fit); fit before "
                               "enable_data_parallel()")
        hp = self.hp
        left = max(int(hp.nr_iter_sphere_fit) - self.sphere_fit_iter, 0)
        n = left if nr_iters is None else min(max(int(nr_iters), 0), left)
        self.model_sdf.train()
        opt = self.optimizer
        for g in opt.param_groups:
            g["lr"] = hp.lr               # constant during the fit: the reference creates its LR scheduler when the fit ends
        gi = [i for i, g in enumerate(opt.param_groups) if g.get("name") == "model_sdf"]
        args = (int(nr_points), float(radius), [float(c) for c in center])
        loss = None
        if self._direct is None:
            self.execution["sphere_fit"] = "torch.autograd (%s)" % self._direct_why
            for _ in range(n):
                loss = self._fit_sphere_autograd(gi, *args)
            return loss
        self.execution["sphere_fit"] = "direct kernel sequence (iteration.py)" + (", CUDA-graph replay" if self._cg is not None else "")
        dev = opt.flat_param.device
        fit = self._fit
        if fit is None:
            fit = self._fit = dict(it_dev=torch.zeros((), device=dev), step_dev=torch.zeros(1, dtype=torch.int32, device=dev), graph=None,
                                   warm=None)
        # device-resident fit iteration and AdamW step count: the same sequence runs eagerly and from the captured graph
        fit["it_dev"].fill_(float(self.sphere_fit_iter))
        step_dev = opt.step_dev if opt.device_step else fit["step_dev"]
        if not opt.device_step:
            step_dev.fill_(opt.step_count)
        opt.sync_hyper()
        opt.zero_grad(set_to_none=False)          # every gradient starts clean; the AdamW sweep re-zeroes the SDF group's
        u01 = (self.fixed_random or {}).get("sphere_fit_u01")
        key = args[:2] + (tuple(args[2]), None if u01 is None else u01.data_ptr(), step_dev.data_ptr())

        def one(dit):
            out = self._direct.sphere_fit(dit, *args)
            opt.step_groups_deferred(gi, step_dev)
            self.model_sdf.fused.repack(advance=(step_dev, fit["it_dev"]))
            return out, self.last

        for _ in range(n):
            dit = DeviceIter(self.sphere_fit_iter, fit["it_dev"])
            if self._cg is None:
                loss = one(dit)[0]
            else:
                loss, self.last = run(self._cg, fit, key, dit, one, keep=lambda: self._direct._fit_ws)
            opt.step_count += 1
            self.sphere_fit_iter += 1
        opt._clean = True
        return loss

    def _fit_sphere_autograd(self, gi, nr_points, radius, center):
        """one sphere-fit iteration in the autograd formulation: loss_sphere_init, loss.backward(), AdamW over the SDF group"""
        opt = self.optimizer
        fused_opt = hasattr(opt, "flat_grad")
        dev = next(self.model_sdf.parameters()).device
        u01 = self.draw("sphere_fit_u01", lambda: torch.rand(3, nr_points, device=dev))
        opt.zero_grad(set_to_none=not fused_opt)        # torch AdamW: parameters without a gradient keep no optimizer state
        loss, l_sdf, l_eik = loss_sphere_init(nr_points, self.aabb, self.model_sdf, self.sphere_fit_iter,
                                              points=self.aabb.rand_points_inside_u01(u01), sphere_radius=radius, sphere_center=center)
        loss.backward()
        if fused_opt:
            opt.step(groups=gi)
            if getattr(self.model_sdf, "fused", None) is not None:
                self.model_sdf.fused.repack()          # raw-pointer updates do not bump tensor versions
        else:
            opt.step()
        self.sphere_fit_iter += 1
        self.last = dict(sphere_fit_terms=torch.stack([l_sdf.detach(), l_eik.detach()]))
        return loss.detach()

    # ------------------------------------------------------------------------------------ CUDA-graph replay
    def enable_cuda_graph(self, warmup_steps=3):
        """Run the iteration from CUDA graphs: sync-free static-capacity containers, device-resident pcg32 generators,
        iteration number and AdamW step count, so that one captured (losses + backward) graph and one (optimizer) graph
        replay until the Python control flow of the iteration would change (DeviceIter validity range).
        The first `warmup_steps` iterations run eagerly (on the capture stream) with the same static shapes."""
        if not hasattr(self.optimizer, "flat_grad"):
            raise RuntimeError("CUDA-graph mode needs the flat-buffer optimizer (optimizer='fused')")
        sampler_graph_mode(True, (OccupancyGrid.m_rng, RaySampler.m_rng, VolumeRendering.m_rng))
        opt = self.optimizer
        opt.device_step = True
        dev = opt.flat_param.device
        opt.step_dev = torch.full((1,), opt.step_count, dtype=torch.int32, device=dev)
        opt.sync_hyper()
        self._cg = dict(warm=int(warmup_steps), fb=None, opt={}, occ=None, it_dev=torch.zeros((), device=dev), it_host=None,
                        stream=torch.cuda.Stream(device=dev), launches=0, captures=0,      # captures: the sphere fit's (graphs.run)
                        # the parameter-free head of the iteration (ray generation + occupancy sampling) is a graph of its own on this stream:
                        # it runs beside the previous iteration's optimizer step (see _step_graphed)
                        stream_a=torch.cuda.Stream(device=dev), ev_fb=None, split=(self._direct is not None))

    def disable_cuda_graph(self):
        """back to eager iterations with exactly-sized containers (host sync per compaction, like the reference)"""
        if self._cg is None:
            return
        torch.cuda.synchronize()
        sampler_graph_mode(False, (OccupancyGrid.m_rng, RaySampler.m_rng, VolumeRendering.m_rng))
        self.optimizer.device_step = False
        self.optimizer.step_dev = None
        self._cg = None
        self._fit = None                # its graph slot reads the step count just dropped

    def _sync_device_iter(self):
        cg = self._cg
        if cg["it_host"] != self.iter_nr:
            cg["it_dev"].fill_(float(self.iter_nr))
            cg["it_host"] = self.iter_nr

    def step_from_reel(self, tensor_reel, pixel_indices, image_indices, update_occupancy=None, optimizer_step=True, inputs_ready=False,
                       loss_to_host=False):
        """one iteration from (pixel, image) indices into a TensorReel: ray generation (PermutoSDF.rays_from_reel_indices) + step.
        Under CUDA-graph replay the indices are the graph's inputs -- host (pinned) or device int32 tensors, copied straight into the
        static buffers -- and the ray-generation kernel is part of the replayed graph."""
        make_rays = lambda pix, img: PermutoSDF.rays_from_reel_indices(tensor_reel, pix, img)
        if self._cg is None:
            dev = self.optimizer.flat_param.device if hasattr(self.optimizer, "flat_param") else torch.device("cuda", torch.cuda.current_device())
            with torch.no_grad():
                o, d, gt, gm, idx = make_rays(pixel_indices.to(dev, non_blocking=True), image_indices.to(dev, non_blocking=True))
            return self.step(o, d, gt, gm, idx, update_occupancy=update_occupancy, optimizer_step=optimizer_step)
        self.model_sdf.train(); self.model_rgb.train()
        return self._step_graphed(pixel_indices, image_indices, None, None, None, update_occupancy, optimizer_step, make_rays=make_rays,
                                  inputs_ready=inputs_ready, loss_to_host=loss_to_host)

    def _step_graphed(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, update_occupancy, optimizer_step, make_rays=None,
                      inputs_ready=False, loss_to_host=False):
        cg = self._cg
        it = self.iter_nr
        if self._dp is not None:
            # data-parallel runs: keep the host at most TWO iterations ahead of the GPU (wait for the end of the forward/backward graph of
            # the iteration before the previous one). With the host free to queue many iterations of graph replays + eagerly launched
            # cross-rank barrier / peer-step kernels on two streams, data-parallel step times were unstable from run to run (the process
            # spun), while the end-to-end path -- which reads the loss every step and so never runs ahead -- was steady. Two iterations of
            # queued work keep the GPU fed; the wait costs nothing then.
            hist = cg.setdefault("ev_hist", [])
            if len(hist) >= 2:
                hist[-2].synchronize()
        self._sync_device_iter()
        # with make_rays the graph inputs are (pixel indices, image indices) and ray generation is captured with the iteration
        inputs = [ray_origins, ray_dirs] if make_rays is not None else [ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices]
        hp = self.hp
        # by-value constants of the captured kernels: a schedule edit (eikonal 0.04 -> 0.01 at iter_start_reduce_curv) re-captures
        consts = (hp.eikonal_weight, hp.curvature_weight, hp.mask_weight, hp.offsurface_weight, hp.lipshitz_weight)
        shapes = (make_rays is not None, consts) + tuple(None if t is None else (tuple(t.shape), t.dtype) for t in inputs)
        fb = cg["fb"]
        valid = fb is not None and fb["shapes"] == shapes and fb["lo"] <= it < fb["hi"]
        cur = torch.cuda.current_stream()
        if not valid and cg["warm"] > 0:
            # eager iteration with the static shapes, on the capture stream (lazy library state initialises there)
            cg["warm"] -= 1

            def eager():
                args = inputs
                if make_rays is not None:
                    with torch.no_grad():
                        args = make_rays(*[t.to(cg["it_dev"].device, non_blocking=True) for t in inputs])
                self.optimizer.zero_grad(set_to_none=False)
                loss = self.forward_backward(*args, DeviceIter(it, cg["it_dev"]))
                self._dp_join_backward()
                return loss
            loss = on_stream(cg["stream"], eager)
        else:
            if not valid:
                fb = cg["fb"] = self._capture_forward_backward(inputs, shapes, it, make_rays)
            if fb.get("graph_a") is not None:
                # Two graphs. A (inputs -> rays -> occupancy samples) reads no network parameter: it is replayed on its own stream and only
                # waits for the END OF THE PREVIOUS ITERATION'S forward/backward graph (whose kernels read the containers A overwrites) and
                # occupancy refresh -- not for the previous optimizer step, which is still running on the current stream: the HBM-bound
                # AdamW sweep and the latency-bound occupancy march overlap. B (everything else) follows on the current stream.
                side = cg["stream_a"]
                if cg["ev_fb"] is not None:
                    side.wait_event(cg["ev_fb"])
                else:
                    side.wait_stream(cur)
                if not inputs_ready and any(t is not None and t.is_cuda for t in inputs):
                    side.wait_stream(cur)                    # device inputs may have been produced on the current stream just now
                with torch.cuda.stream(side):
                    for dst, src in zip(fb["static"], inputs):
                        if dst is not None:
                            dst.copy_(src, non_blocking=True)
                    fb["graph_a"].replay()
                cur.wait_stream(side)
            else:
                for dst, src in zip(fb["static"], inputs):
                    if dst is not None:
                        dst.copy_(src, non_blocking=True)
            self.optimizer.zero_grad(set_to_none=False)     # no-op unless a previous iteration skipped its optimizer step
            fb["graph"].replay()
            self.last = fb["last"]
            loss = fb["loss"]
            for m in (self.model_sdf, self.model_rgb, self.model_bg):
                if m is not None:
                    m.last_iter_nr = it
        if loss_to_host:
            # 4-byte copy + event right behind the forward/backward graph: the host reads the loss without waiting for the optimizer step
            if cg.get("loss_host") is None:
                cg["loss_host"], cg["ev_loss"] = torch.zeros(1).pin_memory(), torch.cuda.Event()
            cg["loss_host"].copy_(loss.detach().reshape(1), non_blocking=True)
            cg["ev_loss"].record(torch.cuda.current_stream())
            loss = HostLoss(cg["loss_host"], cg["ev_loss"], loss)
        if update_occupancy is None:
            update_occupancy = (it % 8 == 0)
        if update_occupancy and self.hp.use_occupancy_grid:
            self._update_occupancy_graphed(it)
        if self.hp.adaptive_nr_rays:
            self.adapt_nr_rays(int(self.last["nr_samples_dev"].item()))     # the reference's loop reads the count every iteration too
        if cg.get("split"):
            ev = cg["ev_fb"] if cg["ev_fb"] is not None else torch.cuda.Event()
            ev.record(torch.cuda.current_stream())          # forward/backward (+ occupancy refresh) of this iteration are queued up to here
            cg["ev_fb"] = ev
        if self._dp is not None:
            e = torch.cuda.Event()
            e.record(torch.cuda.current_stream())
            hist = cg.setdefault("ev_hist", [])
            hist.append(e)
            del hist[:-3]
        self.apply_schedules(it)
        if optimizer_step:
            self.optimizer_step()
        self.iter_nr += 1
        return loss

    def _update_occupancy_graphed(self, it):
        """the occupancy refresh of every 8th iteration (random voxel sample -> fused SDF forward -> grid update,
        train_permuto_sdf.py:386-391) as a third replayed graph: one launch instead of five, same device-resident schedule rule
        (re-captured when the iteration leaves the range for which the captured branches hold)"""
        cg = self._cg
        og = cg.get("occ")
        dit = DeviceIter(it, cg["it_dev"])
        if cg["fb"] is None:                     # warm-up iterations: eager, on the capture stream
            on_stream(cg["stream"], self.update_occupancy, dit)
            return
        if og is None or not (og["lo"] <= it < og["hi"]):
            g, _, launches = capture(cg["stream"], self.update_occupancy, dit, count_launches=True)
            og = cg["occ"] = dict(graph=g, lo=dit.lo, hi=dit.hi, launches=launches)
        og["graph"].replay()
        from ._lib import stats_add_launches
        stats_add_launches(og["launches"])

    def _capture_forward_backward(self, inputs, shapes, it, make_rays=None):
        cg = self._cg
        static = [None if t is None else t.detach().to(cg["it_dev"].device).clone() for t in inputs]
        dit = DeviceIter(it, cg["it_dev"])
        self.optimizer.zero_grad(set_to_none=False)

        def rays():
            if make_rays is None:
                return static
            with torch.no_grad():
                return make_rays(*static)

        def forward_backward(args, pre=None):
            out = self.forward_backward(*args, dit, pre=pre)
            self._dp_join_backward()
            return out

        if cg.get("split") and self._direct is not None:
            # graph A: inputs -> rays -> occupancy samples (no network parameter read); graph B: the rest, sharing A's memory pool
            def head():
                args = rays()
                return args, self._direct.sample_uniform(args[0], args[1])
            g_a, (args, pre), launches_a = capture(cg["stream_a"], head, count_launches=True)
            g, out, launches = capture(cg["stream"], forward_backward, args, pre, pool=g_a.pool(), count_launches=True)
            launches += launches_a
        else:
            g_a = None
            g, out, launches = capture(cg["stream"], lambda: forward_backward(rays()), count_launches=True)
        dp_rgb = bool(self._dp.pop("rgb_reduced", False)) if getattr(self, "_dp", None) is not None else False
        cg["occ"] = None               # the refresh graph reads tensors of the iteration graph (last inv_s): capture it again
        cg["ev_fb"] = None             # the first replay waits for everything queued so far
        return dict(graph=g, graph_a=g_a, static=static, loss=out, last=self.last, shapes=shapes, lo=dit.lo, hi=dit.hi, launches=launches,
                    dp_rgb_reduced=dp_rgb)

    def _optimizer_step_graphed(self, grad_scale, allreduce=False):
        """the optimizer half of a replayed iteration: (data-parallel: bucketed all-reduce overlapped with AdamW,) AdamW, weight re-pack,
        iteration++ -- captured once per (grad_scale, collective layout) and replayed; NCCL collectives are part of the graph"""
        cg = self._cg
        dp = getattr(self, "_dp", None)
        self.optimizer.sync_hyper()     # lr / weight_decay edits since the last replay -> device (outside any capture)
        if dp is not None:
            rgb_done = cg["fb"]["dp_rgb_reduced"] if cg["fb"] is not None else dp.pop("rgb_reduced", False)
        else:
            rgb_done = False

        def work():
            deferred = False
            if dp is not None:
                self._dp_optimizer_step(rgb_done)
            else:
                if allreduce:
                    import torch.distributed as dist
                    dist.all_reduce(self.optimizer.flat_grad, op=dist.ReduceOp.SUM)
                # every group in one launch; the step counter is advanced by the re-pack below (2 launches instead of 7)
                deferred = self.optimizer.step(grad_scale=grad_scale, defer_counter=True, leave_room=bool(cg.get("split"))) is True
            if deferred:
                self.model_sdf.fused.repack(advance=(self.optimizer.step_dev, cg["it_dev"]))
            else:
                self.model_sdf.fused.repack(advance=(None, cg["it_dev"]))

        if cg["fb"] is None:            # still in the eager warm-up iterations
            on_stream(cg["stream"], work)
        elif dp is not None and dp["mode"] == "peer":
            # the cross-rank barriers of the peer-memory step are launched eagerly, right behind the replayed iteration graph (a handful
            # of launches; the host is far ahead of the GPU)
            work()
        else:
            key = (grad_scale, allreduce, dp is not None, rgb_done)
            og = cg["opt"].get(key)
            if og is None:
                g, _, launches = capture(cg["stream"], work, count_launches=True)
                self.optimizer.step_count -= 1          # capture records, it does not run
                og = cg["opt"][key] = dict(graph=g, launches=launches)
            og["graph"].replay()
            self.optimizer.step_count += 1
        if cg["it_host"] is not None:
            cg["it_host"] += 1          # the device-resident iteration number was advanced with the optimizer

    def graph_launches_per_step(self):
        """kernels of this library inside one replayed iteration (counted while capturing)"""
        cg = self._cg
        if cg is None or cg["fb"] is None:
            return None
        return cg["fb"]["launches"] + sum(o["launches"] for o in cg["opt"].values())

    def optimizer_step(self, grad_scale=1.0, allreduce=False):
        """AdamW (+ weight re-pack). After enable_data_parallel() the gradient all-reduce and the 1/world mean are part of the step."""
        if self._cg is not None:
            return self._optimizer_step_graphed(float(grad_scale), bool(allreduce))
        dp = getattr(self, "_dp", None)
        if dp is not None:
            self._dp_optimizer_step(dp.pop("rgb_reduced", False))
            if getattr(self.model_sdf, "fused", None) is not None:
                self.model_sdf.fused.repack()
            return
        if allreduce:
            import torch.distributed as dist
            dist.all_reduce(self.optimizer.flat_grad, op=dist.ReduceOp.SUM)
        if hasattr(self.optimizer, "flat_grad"):
            self.optimizer.step(grad_scale=grad_scale)
            if getattr(self.model_sdf, "fused", None) is not None:
                self.model_sdf.fused.repack()      # raw-pointer updates do not bump tensor versions
        else:
            if grad_scale != 1.0:
                for p in self.params:
                    if p.grad is not None:
                        p.grad.mul_(grad_scale)
            self.optimizer.step()
