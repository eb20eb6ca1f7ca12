"""Direct (autograd-free) training iteration: forward, losses and backward of train_permuto_sdf.py:311-422 (`--with_mask`) as an
explicit sequence of C-ABI calls.

`Trainer.losses()` + `loss.backward()` formulate the iteration with torch.autograd around the fused kernels: correct, but between the
big kernels autograd and the schedule / loss arithmetic spend ~70 one-block launches per iteration (zero-fills, `mul`, `add`, `exp`,
`sum`, per-layer Lipschitz normalisation, calibration, gradient accumulation) -- a large share of the step time even inside a
CUDA graph. Here the same mathematics is issued directly:

    sampling (occupancy grid + 2 importance rounds)                                    unchanged, no gradients
    psdf_iter_scalars                   cos-anneal ratio, inv_s = exp(10 forced_variance), curvature ramp          1 launch
    torch.rand + psdf_sphere_rand_points_inside_u01      off-surface points                                         2
    psdf_sdf_fused_forward_multi        sdf, d sdf/dx, geom at the samples + sdf at the off-surface points          1
    psdf_lipschitz_pack4                Lipschitz normalisation of the 4 colour matrices + operand packing          1
    psdf_rgb_fused_forward              raw colour                                                                   1
    psdf_neus_head_loss_forward         calibration + sigmoid + NeuS compositing + per-ray loss terms               1
    torch.randn + psdf_curvature_shift_points + psdf_sdf_fused_forward   curvature pass                             3
    psdf_loss_terms                     every reduction, the weighted total, the off-surface gradient seed           1
    psdf_neus_head_loss_backward        d / d {sdf, grad, raw colour, shifted grad}, calibration gradients, tail zero-fill   1
    psdf_rgb_fused_backward_acc         colour network backward, d / d sdf-gradient accumulated in place            2 kernels
    psdf_lipschitz_backward4            4 normalisation backwards (+ Lipschitz-bound loss), into .grad               1
    psdf_sdf_fused_backward_multi       the three SDF sample sets                                                    1

Parameter gradients are accumulated straight into the flat-buffer optimizer's `.grad` views (which the AdamW kernel leaves zeroed).
Every formula is the one of the autograd path; `tests/test_direct_iteration_gpu.py` compares loss and all parameter gradients of the
two formulations."""
import ctypes

import torch

from ._lib import call
from .models import DeviceIter
from .permuto_sdf import RaySamplesPacked


class DirectIteration:
    N_OFF = 1024          # off-surface points per iteration (train_permuto_sdf.py:374-378)

    def __init__(self, trainer):
        self.tr = trainer
        self._ws = None
        self._ws_key = None
        self._fixed = None
        self._scal_params = None

    # ------------------------------------------------------------------------------------------ applicability
    @staticmethod
    def unsupported_reason(tr):
        hp = tr.hp
        if not hp.with_mask or tr.model_bg is not None:
            return "background model (no --with_mask) runs on the autograd formulation"
        if not tr.fused_render:
            return "fused_render is off"
        if getattr(tr.model_sdf, "fused", None) is None or not getattr(tr.model_sdf, "fused_training", False):
            return "the SDF model is not on the fused training kernels"
        if getattr(tr.model_rgb, "fused", None) is None:
            return "the colour model is not on the fused kernels"
        if not hasattr(tr.optimizer, "flat_grad"):
            return "needs the flat-buffer optimizer (gradients accumulate into persistent .grad views)"
        if not hp.do_importance_sampling or not hp.use_occupancy_grid:
            return "needs occupancy-grid sampling with importance resampling"
        return None

    # ------------------------------------------------------------------------------------------ persistent buffers
    def _fixed_workspace(self, dev):
        """buffers whose size does not depend on the sample count (used by the part of the iteration that runs beside the sampling)"""
        if self._fixed is not None and self._fixed["dev"] == str(dev):
            return self._fixed
        fr = self.tr.model_rgb.fused
        dims = [fr.in_dim] + fr.h + [3]
        sizes = [dims[l + 1] * dims[l] for l in range(4)]
        gweff = torch.zeros(sum(sizes), device=dev)          # d loss / d W_eff: accumulated by k_rgb_fused_backward (per-tile reductions), reset by psdf_lipschitz_backward4
        offs = [0, sizes[0], sizes[0] + sizes[1], sizes[0] + sizes[1] + sizes[2]]
        f = lambda *s: torch.empty(*s, device=dev)
        self._fixed = dict(dev=str(dev), off_pts=f(self.N_OFF, 3), sdf_off=f(self.N_OFF, 1), g_off=f(self.N_OFF, 1),
                           acc=torch.zeros(8, device=dev), loss=torch.zeros(1, device=dev), terms=torch.zeros(12, device=dev),
                           scal=torch.zeros(8, device=dev),
                           gweff=[gweff[offs[l]:offs[l] + sizes[l]].view(dims[l + 1], dims[l]) for l in range(4)],
                           stream=torch.cuda.Stream(device=dev))
        return self._fixed

    def _workspace(self, N, R, dev):
        key = (N, R, str(dev))
        if self._ws_key == key:
            return self._ws
        tr = self.tr
        fs, fr = tr.model_sdf.fused, tr.model_rgb.fused
        f = lambda *s: torch.empty(*s, device=dev)
        from ._lib import load_library
        lib = load_library()
        ws = dict(self._fixed_workspace(dev))
        ws.update(
            sdf=f(N, 1), grad=f(N, 3), geom=f(N, fs.out_dim - 1), x_raw=f(N, 3),
            shifted=f(N, 3), sdf_s=f(N, 1), grad_s=f(N, 3),
            alpha=f(N), T=f(N), pred=f(R, 3), wsum=f(R, 1), bgT=f(R, 1), ray_loss=f(R, 3),
            g_sdf=f(N, 1), g_grad=f(N, 3), g_x=f(N, 3), g_grad_s=f(N, 3), g_geom=f(N, fs.out_dim - 1),
            rgb_ws=torch.empty(int(lib.psdf_rgb_fused_backward_workspace_bytes(N)), dtype=torch.uint8, device=dev),
            sdf_ws=torch.empty(int(lib.psdf_sdf_fused_backward_multi_workspace_bytes(N, N, self.N_OFF)), dtype=torch.uint8, device=dev),
        )
        self._ws, self._ws_key = ws, key
        return ws

    def _scalars(self, it, ws):
        """cos-anneal ratio [0], inv_s unclipped [1] / clipped [2], curvature ramp [3] from the (device-resident) iteration"""
        hp = self.tr.hp
        if self._scal_params is None:
            P = (ctypes.c_float * 16)(0.0, float(hp.forced_variance_finish_iter), 0.0, 1.0,
                                      0.0, float(hp.forced_variance_finish_iter), 0.3, float(hp.forced_variance_finish),
                                      0.0, float(hp.forced_variance_finish_iter), 0.3, float(hp.forced_variance_finish),
                                      float(hp.iter_start_reduce_curv), float(hp.iter_finish_reduce_curv), 1.0, 0.0)
            K = (ctypes.c_int * 4)(0, 1, 2, 0)
            self._scal_params = (P, K)
        P, K = self._scal_params
        it_dev = it.dev if isinstance(it, DeviceIter) else None
        call("psdf_iter_scalars", 4, ctypes.addressof(P), ctypes.addressof(K), it_dev, float(int(it)), ws["scal"])
        return ws["scal"]

    # ------------------------------------------------------------------------------------------ the iteration
    def sample_uniform(self, ray_origins, ray_dirs):
        """Part A of the iteration: bounding-sphere intersection and occupancy-grid sampling (train_permuto_sdf.py:111-135). It reads no
        network parameter, so under CUDA-graph replay it is a graph of its own that runs beside the previous iteration's optimizer step
        (Trainer._step_graphed). One sphere intersection serves sampling, resampling and the hit mask."""
        tr = self.tr
        hp = tr.hp
        with torch.no_grad():
            _, t_entry, _, t_exit, does_hit = tr.aabb.ray_intersection(ray_origins, ray_dirs)
            jitter = tr.model_sdf.training if getattr(hp, "jitter_samples", None) is None else bool(hp.jitter_samples)
            fg = tr.occupancy_grid.compute_samples_in_occupied_regions(ray_origins, ray_dirs, t_entry, t_exit, hp.min_dist_between_samples,
                                                                       hp.max_nr_samples_per_ray, jitter).compact_to_valid_samples()
        return dict(t_exit=t_exit, does_hit=does_hit, fg=fg, jitter=jitter)

    def run(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, it, pre=None):
        """forward + losses + backward; parameter gradients land in the optimizer's .grad views. -> detached 0-d loss tensor.
        pre: result of sample_uniform() for these rays when it already ran (as its own graph)"""
        from .train import importance_sampling_sdf_model
        tr = self.tr
        hp = tr.hp
        m_sdf, m_rgb, cal = tr.model_sdf, tr.model_rgb, tr.model_colorcal
        fs, fr = m_sdf.fused, m_rgb.fused
        dev = ray_origins.device
        R = ray_origins.shape[0]
        static = RaySamplesPacked.static_capacity
        # Python control flow on the iteration (narrows the validity range of a captured graph, DeviceIter)
        curv_on = it < hp.iter_finish_reduce_curv
        lip_on = it >= hp.iter_start_reduce_curv
        if pre is None:
            pre = self.sample_uniform(ray_origins, ray_dirs)
        t_exit, does_hit, fg, jitter = pre["t_exit"], pre["does_hit"], pre["fg"], pre["jitter"]
        n_off = self.N_OFF
        L = fr.layers
        c = m_rgb.mlp.lipshitz_bound_per_layer
        with torch.no_grad():
            # ---------------- what does not depend on the samples runs on a forked stream beside the importance-sampling chain (a parallel
            # branch of the captured graph): schedule scalars, off-surface points, Lipschitz normalisation + packing of the colour weights
            fx = self._fixed_workspace(dev)
            cur, side = torch.cuda.current_stream(), fx["stream"]
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                scal = self._scalars(it, fx)
                u01 = tr.draw("offsurface_u01", lambda: torch.rand(3, n_off, device=dev))
                call("psdf_sphere_rand_points_inside_u01", n_off, tr.aabb.m_radius, u01, fx["off_pts"])
                call("psdf_lipschitz_pack4", fr.in_dim, *fr.h, 3, L[0].weight.detach(), L[0].bias.detach(), c[0].detach(), L[1].weight.detach(),
                     L[1].bias.detach(), c[1].detach(), L[2].weight.detach(), L[2].bias.detach(), c[2].detach(), L[3].weight.detach(),
                     L[3].bias.detach(), c[3].detach(), fr.blob)
            if fg.samples_pos.shape[0] != 0:
                fg = importance_sampling_sdf_model(m_sdf, fg, ray_origins, ray_dirs, t_exit, it, hp.nr_samples_imp_sampling, jitter=jitter)
            n_mean = None
            if getattr(hp, "dp_world", 1) > 1:
                import torch.distributed as dist
                n_sum = fg.cur_nr_samples.to(torch.int32).clone()
                dist.all_reduce(n_sum, op=dist.ReduceOp.SUM)
                W = int(hp.dp_world)
                n_mean = fg.dp_mean_nr_samples = torch.div(n_sum + W // 2, W, rounding_mode="floor").to(torch.int32).clamp(min=1)
            cur.wait_stream(side)                # join the forked branch
            N = fg.samples_pos.shape[0]
            if N == 0:
                return None                      # no sample at all (eager mode only): the caller takes the autograd formulation
            ws = self._workspace(N, R, dev)
            n_valid = fg.cur_nr_samples if static else None
            cos_dev, inv_s = scal[0:1], scal[1:2]
            m_rgb.volume_renderer_neus.last_inv_s = scal[2:3]
            m_rgb.volume_renderer_neus.deviation_network.last_variance = None
            # ---------------- SDF at the samples (+ off-surface points)
            if fs._versions != fs._cur_versions():
                fs.repack()
            enc = m_sdf.encoding
            m_sdf.last_iter_nr = int(it)
            win = m_sdf.window(it).view(-1).contiguous()
            pos = fg.samples_pos
            sdf_args = (enc.nr_levels, enc.capacity, enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(), win,
                        enc.concat_points_scaling, fs.hidden, fs.out_dim, fs.blob)
            call("psdf_sdf_fused_forward_multi", *sdf_args, N, pos, ws["sdf"], ws["grad"], ws["geom"], n_off, ws["off_pts"], ws["sdf_off"],
                 None, None)
            # ---------------- colour network (weights normalised + packed on the forked branch)
            enc_c = m_rgb.encoding
            win_c = fr._window(it)
            rgb_args = (N, enc_c.nr_levels, enc_c.capacity, pos, fg.samples_dirs, ws["grad"], ws["geom"], ws["geom"].shape[1],
                        enc_c.lattice_values.detach(), enc_c.scale_factor, enc_c.shift_tensor(), win_c, enc_c.concat_points_scaling, *fr.h, fr.blob)
            call("psdf_rgb_fused_forward", *rgb_args, ws["x_raw"])
            # ---------------- compositing + per-ray losses (colour head folded in)
            hit = does_hit.reshape(-1)
            mask = gt_mask.detach().reshape(-1).float().contiguous() if (hp.with_mask and gt_mask is not None) else None
            gt = gt_rgb.detach().contiguous()
            if cal is not None and img_indices is not None:
                img = img_indices.detach().reshape(-1)
                img = img if img.dtype == torch.int32 else img.to(torch.int32)
                head = (img, cal.weight_delta.detach(), cal.bias.detach(), int(cal.idx_with_fixed_calib))
            else:
                head = (None, None, None, -1)
            sdf_flat = ws["sdf"].view(-1)
            neus_in = (*fg._rsp(), sdf_flat, ws["grad"], ws["x_raw"], fg.samples_dirs, fg.samples_dt, inv_s, 0.0, cos_dev, gt, mask, hit, *head)
            call("psdf_neus_head_loss_forward", *neus_in, ws["alpha"], ws["T"], None, ws["pred"], ws["wsum"], ws["bgT"], ws["ray_loss"])
            # ---------------- curvature pass (models.py:261-294)
            gs = None
            if curv_on:
                rnd = tr.draw("curvature_dirs", lambda: torch.randn_like(pos))
                call("psdf_curvature_shift_points", N, pos, ws["grad"], rnd, 1e-4, ws["shifted"])
                call("psdf_sdf_fused_forward", N, enc.nr_levels, enc.capacity, ws["shifted"], enc.lattice_values.detach(), enc.scale_factor,
                     enc.shift_tensor(), win, enc.concat_points_scaling, fs.hidden, fs.out_dim, fs.blob, ws["sdf_s"], ws["grad_s"], None)
                gs = ws["grad_s"]
            # ---------------- all loss terms
            w_mask = float(hp.mask_weight) if mask is not None else 0.0
            w_curv = float(hp.curvature_weight) if curv_on else 0.0
            w_lip = float(hp.lipshitz_weight) if lip_on else 0.0
            c_rgb, c_mask = 1.0 / (3.0 * R), w_mask / R
            call("psdf_loss_terms", N, n_valid, n_mean, ws["grad"], gs, R, ws["ray_loss"], n_off, ws["sdf_off"].view(-1), ws["g_off"].view(-1),
                 c_rgb, c_mask, float(hp.eikonal_weight), w_curv, scal[3:4], float(hp.offsurface_weight), w_lip,
                 c[0].detach(), c[1].detach(), c[2].detach(), c[3].detach(), ws["acc"], ws["loss"], ws["terms"])
            # ================= backward
            n_cnt = n_mean if n_mean is not None else n_valid
            scale_eik = float(hp.eikonal_weight) if n_cnt is not None else float(hp.eikonal_weight) / max(N, 1)
            g_wd = cal.weight_delta.grad if head[1] is not None else None
            g_cb = cal.bias.grad if head[1] is not None else None
            call("psdf_neus_head_loss_backward", *neus_in, ws["alpha"], ws["T"], ws["pred"], ws["wsum"], ws["bgT"], c_rgb, c_mask, scale_eik, n_cnt,
                 gs, w_curv, scal[3:4], N, n_valid, ws["g_sdf"].view(-1), ws["g_grad"], ws["g_x"], ws["g_grad_s"] if gs is not None else None,
                 g_wd, g_cb)
            gW = ws["gweff"]
            call("psdf_rgb_fused_backward_acc", *rgb_args, ws["g_x"], enc_c.lattice_values.grad, ws["g_grad"], ws["g_geom"], ws["rgb_ws"],
                 gW[0], gW[1], gW[2], gW[3], L[0].bias.grad, L[1].bias.grad, L[2].bias.grad, L[3].bias.grad)
            if getattr(fr, "after_backward", None) is not None:
                fr.after_backward()          # data-parallel (NCCL overlap mode): the colour hash-table gradient is final
            lip_args = []
            for l in range(4):
                lip_args += [L[l].weight.detach(), c[l].detach(), gW[l], L[l].weight.grad, c[l].grad]
            call("psdf_lipschitz_backward4", fr.in_dim, *fr.h, 3, *lip_args, w_lip)
            segs = [N, pos, ws["g_sdf"].view(-1), ws["g_grad"], ws["g_geom"]]
            segs += [N, ws["shifted"], None, ws["g_grad_s"], None] if gs is not None else [0, None, None, None, None]
            segs += [n_off, ws["off_pts"], ws["g_off"].view(-1), None, None]
            lin = fs.lin
            call("psdf_sdf_fused_backward_multi", *sdf_args, *segs, enc.lattice_values.grad, ws["sdf_ws"],
                 lin[0].weight.grad, lin[1].weight.grad, lin[2].weight.grad, lin[3].weight.grad,
                 lin[0].bias.grad, lin[1].bias.grad, lin[2].bias.grad, lin[3].bias.grad)
        t = ws["terms"]
        tr.last = dict(loss_rgb=t[8], loss_eikonal=t[9], loss_curvature=t[3], nr_samples=N, nr_samples_dev=fg.cur_nr_samples, fg=fg,
                       terms=t)
        return ws["loss"].view(())
