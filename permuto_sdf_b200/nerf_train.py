"""NeRF training on the fused kernels: the loop of train_nerf.py:131-226 as a direct, graph-replayable kernel sequence.

Each iteration of the reference refreshes the 64^3 occupancy grid from density every 8th iteration, draws 512 rays, samples them
(occupancy-grid samples for the foreground NerfHash(3), 32 NeRF++ samples per ray for the background NerfHash(4) of scenes without
masks), composites both, applies the rgb loss (+ 0.1 BCE of the weights sum with masks) and runs AdamW. `NerfTrainer.step()` issues the
same mathematics without autograd:

    ray-sphere intersection + train.create_samples       the hit mask, occupancy samples (compacted), background samples
    psdf_bg_mlp_pack x 2                                  operand blobs of both networks
    coarse-to-fine windows                                from the device-resident iteration (element-wise torch ops while they ramp)
    psdf_nerf_fused_forward(3)                            foreground colour (linear) and density
    psdf_nerf_fused_forward(4) + psdf_nerf_bg_composite_forward      background colour per ray (no mask only)
    psdf_nerf_loss_forward                                calibration, sigmoid, compositing, background blend, loss
    psdf_nerf_loss_backward                               d loss / d {colour, density, background colour}, calibration gradients
    psdf_nerf_bg_composite_backward + psdf_nerf_fused_backward(4)    background backward (no mask only)
    psdf_nerf_fused_backward(3)                           foreground backward into the optimizer's .grad views
    psdf_adamw_multi_step                                 AdamW over every parameter
    step count + iteration                                two in-place adds on the device

and, every 8th iteration before the rays, the refresh: compute_random_sample_of_grid_points(256^2, True), the fused D = 3 forward at the
points (zero directions, colour discarded) and psdf_occ_update_with_density(decay 0.7, threshold 1e-3).

The step count and iteration live on the device in eager runs too, so an eager run and one replayed from captured CUDA graphs
(`enable_cuda_graph()`) give the same bits in deterministic mode. The autograd formulation of train_nerf.py (`NerfHash`,
`VolumeRenderingNerf`, the torch losses, `loss.backward()`) is the fallback and the yardstick of the tests and of
tools/bench_nerf_train.py."""
import os

import torch
import torch.nn.functional as F

from ._lib import call, load_library
from .models import Colorcal, DeviceIter, NerfHash, map_range_val
from .permuto_sdf import OccupancyGrid, PermutoSDF, RaySampler, RaySamplesPacked, Sphere

_INT32_MAX = 2 ** 31 - 1
MASK_WEIGHT = 0.1                                  # train_nerf.py:182
OCC_NR_POINTS, OCC_DECAY, OCC_THRESH, OCC_EVERY = 256 * 256, 0.7, 1e-3, 8      # train_nerf.py:159-163


class NerfHyperParams:
    """train_nerf.py:45-56"""
    lr = 1e-3
    iter_finish_training = 200000
    use_occupancy_grid = True
    nr_samples_bg = 32
    min_dist_between_samples = 0.0001
    max_nr_samples_per_ray = 64
    use_color_calibration = True
    nr_rays = 512
    foreground_nr_iters_for_c2f = 1
    background_nr_iters_for_c2f = 10000


def nerf_loss(gt_rgb, pred_rgb, does_ray_intersect_box, weights_sum=None, gt_mask=None):
    """train_nerf.py:176-182 -> (loss, loss_rgb, loss_mask or None)"""
    loss_rgb = ((gt_rgb - pred_rgb) ** 2 * does_ray_intersect_box * 1.0).mean()
    if gt_mask is None:
        return loss_rgb, loss_rgb, None
    loss_mask = F.binary_cross_entropy(weights_sum.clip(1e-3, 1.0 - 1e-3), gt_mask)
    return loss_rgb + loss_mask * MASK_WEIGHT, loss_rgb, loss_mask


def _check_levels(nr_levels):
    if nr_levels % 4 != 0 or nr_levels > 28 or nr_levels < 4:
        raise RuntimeError("NerfTrainer: nr_levels must be a multiple of 4 between 4 and 28 (the fused NerfHash kernels take 2L + 4 <= 64 "
                           "encoder columns in whole 8-column cores), got %d" % nr_levels)


class NerfTrainer:
    """The state and the loop of train_nerf.py: NerfHash(3) foreground, NerfHash(4) background (scenes without masks), Colorcal(nr_images, 0),
    OccupancyGrid(64, 1.0, [0,0,0]) inside the bounding Sphere(0.5, [0,0,0]), one AdamW over every parameter (betas (0.9, 0.99), eps 1e-15,
    no weight decay, constant lr).

    optimizer "fused" (flat-buffer AdamW kernel) or "adamw" (torch.optim.AdamW). direct: None = the direct kernel sequence whenever the
    configuration allows it, True = require it, False = the autograd formulation. deterministic: the library's deterministic mode for this
    device (order-independent reductions). `execution` records which path runs and why."""

    def __init__(self, nr_images, with_mask, nr_levels=24, capacity=2 ** 18, optimizer="fused", deterministic=False, direct=None, seed=0,
                 hyperparams=None):
        _check_levels(int(nr_levels))
        if optimizer not in ("fused", "adamw"):
            raise RuntimeError("NerfTrainer: optimizer must be 'fused' or 'adamw', got %r" % (optimizer,))
        self.hp = hp = hyperparams or NerfHyperParams()
        self.with_mask = bool(with_mask)
        torch.manual_seed(seed)
        dev = torch.device("cuda", torch.cuda.current_device())
        self.aabb = Sphere(0.5, [0, 0, 0])
        self.model = NerfHash(3, self.aabb, hp.foreground_nr_iters_for_c2f, nr_levels, capacity).to(dev)
        self.model_bg = None if self.with_mask else NerfHash(4, self.aabb, hp.background_nr_iters_for_c2f, nr_levels, capacity).to(dev)
        self.model_colorcal = Colorcal(int(nr_images), 0) if hp.use_color_calibration else None
        self.occupancy_grid = OccupancyGrid(64, 1.0, [0, 0, 0])
        call("psdf_set_deterministic", 1 if deterministic else 0, nr_levels * capacity * 2, 64 ** 3)
        self.models = [m for m in (self.model, self.model_bg) if m is not None]
        for m in self.models:
            m.enable_fused()
        self.execution = {"networks": "fused wgmma"}
        params = [p for m in self.models for p in m.parameters()]
        if self.model_colorcal is not None:
            params += list(self.model_colorcal.parameters())
        if optimizer == "fused":
            from .optim import FusedAdamW
            self.optimizer = FusedAdamW([{"params": params, "weight_decay": 0.0, "lr": hp.lr, "name": "all"}], betas=(0.9, 0.99), eps=1e-15,
                                        lr=hp.lr)
            for m in self.models:
                m.encoding.grad_in_place = True
        else:
            self.optimizer = torch.optim.AdamW(params, amsgrad=False, betas=(0.9, 0.99), eps=1e-15, weight_decay=0.0, lr=hp.lr)
        why = None
        if direct is False:
            why = "disabled by the caller (direct=False)"
        elif optimizer != "fused":
            why = "needs the flat-buffer optimizer (gradients accumulate into persistent .grad views)"
        elif not hp.use_occupancy_grid:
            why = "needs occupancy-grid sampling (use_occupancy_grid)"
        if why is not None and direct:
            raise RuntimeError("NerfTrainer(direct=True): " + why)
        self.direct = why is None
        self.execution["step"] = "direct kernel sequence (nerf_train.py)" if self.direct else "torch.autograd (%s)" % why
        self.iter_nr = 0
        self.last = {}
        self._ws = {}
        self._dev = None            # device-resident iteration and step count of the direct sequence
        self._cg = None             # CUDA-graph state (enable_cuda_graph)

    # ------------------------------------------------------------------------------------ inputs
    def _check_rays(self, R, has_mask):
        R = int(R)
        hp = self.hp
        if R < 1:
            raise RuntimeError("NerfTrainer.step: needs at least one ray (the loss is a mean over the rays)")
        if R * int(hp.max_nr_samples_per_ray) * 4 > _INT32_MAX or R * int(hp.nr_samples_bg) * 4 > _INT32_MAX:
            raise RuntimeError("NerfTrainer.step: %d rays give more sample rows than the kernels' 32-bit row indexing takes" % R)
        if self.with_mask and not has_mask:
            raise RuntimeError("NerfTrainer(with_mask=True).step: the mask loss needs the ground-truth mask, got none")
        return R

    def _head(self, img_indices):
        cal = self.model_colorcal
        if cal is None or img_indices is None:
            return (None, None, None, -1)
        img = img_indices.detach().reshape(-1)
        img = img if img.dtype == torch.int32 else img.to(torch.int32)
        return (img, cal.weight_delta.detach(), cal.bias.detach(), int(cal.idx_with_fixed_calib))

    # ------------------------------------------------------------------------------------ occupancy refresh
    def _fg_window(self, it):
        return self.model.fused._window(it)

    @torch.no_grad()
    def update_occupancy(self, it):
        """train_nerf.py:159-163: density at a random voxel sample (jittered centres) -> grid update"""
        og = self.occupancy_grid
        pts, idx = og.compute_random_sample_of_grid_points(OCC_NR_POINTS, True)
        density = self._density_fused(pts, it) if self.direct else self._density_autograd_model(pts, it)
        og.update_with_density_random_sample(idx, density, OCC_DECAY, OCC_THRESH)

    def _density_fused(self, pts, it):
        """the full fused D = 3 forward at OCC_NR_POINTS points (zero directions; the colour is discarded) -> density [n,1]"""
        fb, enc = self.model.fused, self.model.encoding
        ws = self._ws.get("occ")
        if ws is None:
            dev = pts.device
            ws = self._ws["occ"] = dict(dirs=torch.zeros(OCC_NR_POINTS, 3, device=dev), rgb=torch.empty(OCC_NR_POINTS, 3, device=dev),
                                        density=torch.empty(OCC_NR_POINTS, 1, device=dev))
        fb.pack(fb.params())
        call("psdf_nerf_fused_forward", 3, OCC_NR_POINTS, enc.nr_levels, enc.capacity, pts, ws["dirs"], enc.lattice_values.detach(),
             enc.scale_factor, enc.shift_tensor(), self._fg_window(it), enc.concat_points_scaling, fb.blob, ws["rgb"], ws["density"])
        return ws["density"]

    def _density_autograd_model(self, pts, it):
        """NerfHash.get_only_density (models.py:520-535) on the per-op encoder"""
        m = self.model
        m.last_iter_nr = int(it)
        window = m.c2f(map_range_val(it, 0.0, m.nr_iters_for_c2f, 0.3, 1.0))
        fd = m.mlp_feat_and_density(m.encoding(pts, window.view(-1)))
        return F.softplus(fd[:, 0:1])

    # ------------------------------------------------------------------------------------ the iteration
    def step(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices):
        """one iteration -> detached 0-d loss (no host sync); last['loss_rgb'], last['loss_mask'] (with masks)"""
        self._check_rays(ray_origins.shape[0], gt_mask is not None)
        return self._iterate((ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices), None)

    def step_from_reel(self, tensor_reel, pixel_indices, image_indices):
        """one iteration from (pixel, image) indices into a TensorReel (PermutoSDF.rays_from_reel_indices, the ray kernel of
        random_rays_from_reel); under CUDA-graph replay ray generation is part of the graph"""
        mask = getattr(tensor_reel, "mask_reel", None)
        self._check_rays(pixel_indices.shape[0], mask is not None and mask.numel() > 0)
        make_rays = lambda pix, img: PermutoSDF.rays_from_reel_indices(tensor_reel, pix, img)
        return self._iterate((pixel_indices, image_indices), make_rays)

    def _iterate(self, inputs, make_rays):
        for m in self.models:
            m.train()
        it = self.iter_nr
        if not self.direct:
            opt = self.optimizer
            fused_opt = hasattr(opt, "flat_grad")
            if it % OCC_EVERY == 0:
                self.update_occupancy(it)
            opt.zero_grad(set_to_none=not fused_opt)
            args = self._rays(inputs, make_rays)
            loss = self._autograd_forward_backward(*args, it)
            opt.step()
            self.iter_nr += 1
            return loss
        opt = self.optimizer
        dev = opt.flat_param.device
        st = self._dev
        if st is None:
            st = self._dev = dict(it_dev=torch.zeros((), device=dev), step_dev=torch.zeros(1, dtype=torch.int32, device=dev))
        st["it_dev"].fill_(float(it))
        st["step_dev"].fill_(opt.step_count)
        opt.sync_hyper()
        opt.zero_grad(set_to_none=False)

        def body(dit, args):
            out = self._direct_forward_backward(*self._rays(args, make_rays), dit)
            opt.step_groups_deferred([0], st["step_dev"])
            st["step_dev"].add_(1)
            st["it_dev"].add_(1.0)
            return out

        with torch.cuda.device(dev):
            if self._cg is None:
                if it % OCC_EVERY == 0:
                    self.update_occupancy(DeviceIter(it, st["it_dev"]))
                loss = body(DeviceIter(it, st["it_dev"]), inputs)
            else:
                if it % OCC_EVERY == 0:
                    self._replay("occ", ("occ",), it, st, lambda dit, _: self.update_occupancy(dit), ())
                key = ("step", make_rays is not None) + tuple(None if t is None else (tuple(t.shape), t.dtype) for t in inputs)
                loss = self._replay("step", key, it, st, body, inputs)
        opt.step_count += 1
        opt._clean = True
        self.iter_nr += 1
        return loss

    def _replay(self, name, key, it, st, fn, inputs):
        """fn(DeviceIter, inputs) eagerly on the capture stream the first time a shape is seen, captured the next time, replayed while the
        iteration stays inside the range over which the captured Python control flow holds (DeviceIter)"""
        cg = self._cg
        g = cg["graphs"].get(name)
        if g is not None and g["key"] == key and g["lo"] <= it < g["hi"]:
            for dst, src in zip(g["static"], inputs):
                if dst is not None:
                    dst.copy_(src, non_blocking=True)
            g["graph"].replay()
            self.last = g["last"]
            return g["out"]
        side, cur = cg["stream"], torch.cuda.current_stream()
        dit = DeviceIter(it, st["it_dev"])
        if cg["warm"].get(name) != key:
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                out = fn(dit, inputs)
            cur.wait_stream(side)
            cg["warm"][name] = key
            return out
        dev = st["it_dev"].device
        static = [None if t is None else t.detach().to(dev).clone() for t in inputs]
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            out = fn(dit, static)
        # the buffers the graph writes stay referenced for as long as the graph lives
        cg["graphs"][name] = dict(graph=graph, key=key, lo=dit.lo, hi=dit.hi, out=out, static=static, last=self.last, bufs=dict(self._ws))
        cg["captures"] += 1
        graph.replay()                     # the capture recorded the work, it did not run it
        return out

    def _rays(self, inputs, make_rays):
        if make_rays is None:
            return inputs
        with torch.no_grad():
            dev = self.aabb.m_center_tensor.device
            return make_rays(inputs[0].to(dev, non_blocking=True), inputs[1].to(dev, non_blocking=True))

    def _samples(self, ray_origins, ray_dirs, jitter):
        from .train import create_samples
        return create_samples(self.with_mask, self.hp, ray_origins, ray_dirs, jitter, self.occupancy_grid, self.aabb)

    def _buffers(self, name, shapes):
        """per-shape device buffers of the direct sequence (fixed while the shapes are: static-capacity containers under graph replay)"""
        dev = self.aabb.m_center_tensor.device
        b = self._ws.get(name)
        if b is None or b["shapes"] != shapes:
            b = dict(shapes=shapes)
            for k, s in shapes:
                if k == "ws":
                    b[k] = torch.empty(*s, dtype=torch.uint8, device=dev)
                else:
                    b[k] = torch.zeros(*s, device=dev) if k.startswith("g_") or k == "acc" else torch.empty(*s, device=dev)
            self._ws[name] = b
        return b

    def _forward_fg(self, fg, it, tag="fg"):
        """the D = 3 network at the foreground samples -> (buffers, network arguments)"""
        fb, enc = self.model.fused, self.model.encoding
        N = fg.samples_pos.shape[0]
        lib = load_library()
        ws = self._buffers(tag, (("x", (N, 3)), ("density", (N, 1)), ("g_xd", (N * 4,)),
                                 ("ws", (int(lib.psdf_bg_fused_backward_workspace_bytes(N)),))))
        fb.pack(fb.params())
        args = (3, N, enc.nr_levels, enc.capacity, fg.samples_pos, fg.samples_dirs, enc.lattice_values.detach(), enc.scale_factor,
                enc.shift_tensor(), self._fg_window(it), enc.concat_points_scaling, fb.blob)
        call("psdf_nerf_fused_forward", *args, ws["x"], ws["density"])
        return ws, args

    def _forward_bg(self, bg, it, head, tag="bg"):
        """the D = 4 network at the background samples and its compositing -> (buffers, network arguments, compositing arguments)"""
        fb, enc = self.model_bg.fused, self.model_bg.encoding
        Nb, R = bg.samples_pos_4d.shape[0], bg.ray_start_end_idx.shape[0]
        lib = load_library()
        ws = self._buffers(tag, (("x", (Nb, 3)), ("density", (Nb, 1)), ("bg_rgb", (R, 3)), ("g_bg_rgb", (R, 3)), ("g_x", (Nb, 3)),
                                 ("g_density", (Nb,)), ("ws", (int(lib.psdf_bg_fused_backward_workspace_bytes(Nb)),))))
        fb.pack(fb.params())
        args = (4, Nb, enc.nr_levels, enc.capacity, bg.samples_pos_4d, bg.samples_dirs, enc.lattice_values.detach(), enc.scale_factor,
                enc.shift_tensor(), fb._window(it), enc.concat_points_scaling, fb.blob)
        call("psdf_nerf_fused_forward", *args, ws["x"], ws["density"])
        comp = (*bg._rsp(), ws["x"], ws["density"].view(-1), bg.samples_dt.view(-1), *head)
        call("psdf_nerf_bg_composite_forward", *comp, ws["bg_rgb"])
        return ws, args, comp

    def _direct_forward_backward(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, it, samples=None):
        """forward, loss and backward of iteration `it` (int or DeviceIter); the parameter gradients are ACCUMULATED into the optimizer's
        .grad views. samples: (foreground, background) containers to use instead of drawing them. -> detached 0-d loss"""
        R = ray_origins.shape[0]
        with torch.no_grad():
            _, _, _, _, hit = self.aabb.ray_intersection(ray_origins, ray_dirs)
            fg, bg = samples if samples is not None else self._samples(ray_origins, ray_dirs, self.model.training)
            head = self._head(img_indices)
            fws, fargs = self._forward_fg(fg, it)
            bws = bargs = comp = None
            if bg is not None:
                bws, bargs, comp = self._forward_bg(bg, it, head)
            lw = self._buffers("loss", (("pred", (R, 3)), ("wsum", (R, 1)), ("bgT", (R, 1)), ("acc", (3,)), ("loss", (1,)), ("terms", (2,))))
            mask = gt_mask.detach().reshape(-1).contiguous() if self.with_mask else None
            N = fg.samples_pos.shape[0]
            loss_in = (*fg._rsp(), fws["x"], fws["density"].view(-1), fg.samples_dt.view(-1), *head, None if bws is None else bws["bg_rgb"],
                       gt_rgb.detach().contiguous(), hit.reshape(-1), mask, MASK_WEIGHT)
            call("psdf_nerf_loss_forward", *loss_in, lw["pred"], lw["wsum"], lw["bgT"], None, lw["acc"], lw["loss"], lw["terms"])
            # ================= backward
            cal = self.model_colorcal
            g_wd = cal.weight_delta.grad if head[1] is not None else None
            g_b = cal.bias.grad if head[1] is not None else None
            g_xd = fws["g_xd"]
            g_xd.zero_()                     # rows outside every ray (the tail of static-capacity containers) get no gradient
            g_x, g_den = g_xd[:3 * N].view(N, 3), g_xd[3 * N:]
            call("psdf_nerf_loss_backward", *loss_in, lw["pred"], lw["wsum"], lw["bgT"], g_x, g_den, None if bws is None else bws["g_bg_rgb"],
                 g_wd, g_b)
            if bws is not None:
                call("psdf_nerf_bg_composite_backward", *comp, bws["g_bg_rgb"], bws["g_x"], bws["g_density"], g_wd, g_b)
                lin = self.model_bg.fused.lin
                call("psdf_nerf_fused_backward", *bargs, bws["g_x"], bws["g_density"], self.model_bg.encoding.lattice_values.grad,
                     bws["ws"], *[l.weight.grad for l in lin], *[l.bias.grad for l in lin])
            lin = self.model.fused.lin
            call("psdf_nerf_fused_backward", *fargs, g_x, g_den, self.model.encoding.lattice_values.grad, fws["ws"],
                 *[l.weight.grad for l in lin], *[l.bias.grad for l in lin])
        t = lw["terms"]
        self.last = dict(loss_rgb=t[0], loss_mask=t[1] if self.with_mask else None, nr_samples=N, nr_samples_dev=fg.cur_nr_samples)
        return lw["loss"].view(())

    def _autograd_forward_backward(self, ray_origins, ray_dirs, gt_rgb, gt_mask, img_indices, it, samples=None):
        """train_nerf.py:166-196 with the same draws: run_net, the losses and loss.backward() (gradients accumulate into .grad)"""
        with torch.no_grad():
            _, _, _, _, hit = self.aabb.ray_intersection(ray_origins, ray_dirs)
        pred_rgb, _, weights_sum, _ = self.run_net(ray_origins, ray_dirs, img_indices, it, samples)
        loss, loss_rgb, loss_mask = nerf_loss(gt_rgb, pred_rgb, hit, weights_sum, gt_mask if self.with_mask else None)
        loss.backward()
        self.last = dict(loss_rgb=loss_rgb.detach(), loss_mask=None if loss_mask is None else loss_mask.detach())
        return loss.detach()

    def run_net(self, ray_origins, ray_dirs, img_indices, it, samples=None):
        """train_nerf.py:61-95 (autograd) -> (pred_rgb, pred_rgb_bg or None, weights_sum, samples_pos)"""
        if samples is not None:
            fg, bg = samples
        else:
            with torch.no_grad():
                fg, bg = self._samples(ray_origins, ray_dirs, self.model.training)
        m, cal = self.model, (self.model_colorcal if img_indices is not None else None)
        rgb, density = m(fg.samples_pos, fg.samples_dirs, it, cal, img_indices, ray_start_end_idx=fg.ray_start_end_idx)
        weights, weights_sum, bg_T = m.volume_renderer_nerf.compute_weights(fg, density.view(-1, 1))
        pred_rgb = m.volume_renderer_nerf.integrate(fg, rgb, weights)
        pred_rgb_bg = None
        if bg is not None:
            mb = self.model_bg
            rgb_bg, density_bg = mb(bg.samples_pos_4d, bg.samples_dirs, it, cal, img_indices, ray_start_end_idx=bg.ray_start_end_idx)
            weights_bg, _, _ = mb.volume_renderer_nerf.compute_weights(bg, density_bg.view(-1, 1))
            pred_rgb_bg = mb.volume_renderer_nerf.integrate(bg, rgb_bg, weights_bg)
            pred_rgb_bg = bg_T.view(-1, 1) * pred_rgb_bg
            pred_rgb = pred_rgb + pred_rgb_bg
        return pred_rgb, pred_rgb_bg, weights_sum, fg.samples_pos

    # ------------------------------------------------------------------------------------ rendering
    @torch.no_grad()
    def render(self, ray_origins, ray_dirs, chunk_size=200 * 200):
        """what train_nerf.run_net_in_chunks computes for these rays (no calibration), on the fused kernels, chunk by chunk:
        -> (pred_rgb [R,3], pred_rgb_bg [R,3] or None (scenes with masks), weights_sum [R,1]). Samples are jittered while the model is in
        training mode, as in run_net: put the trainer in eval() to render a frame. Changes no parameter, .grad, grid or counter; without
        jitter it advances no generator."""
        R = int(ray_origins.shape[0])
        if chunk_size < 1:
            raise RuntimeError("NerfTrainer.render: chunk_size must be at least 1")
        out = [torch.empty(R, 3, device=ray_origins.device), None if self.with_mask else torch.empty(R, 3, device=ray_origins.device),
               torch.empty(R, 1, device=ray_origins.device)]
        head = (None, None, None, -1)
        it = self.iter_nr
        for a in range(0, R, int(chunk_size)):
            b = min(R, a + int(chunk_size))
            o, d = ray_origins[a:b].contiguous(), ray_dirs[a:b].contiguous()
            fg, bg = self._samples(o, d, self.model.training)
            fws, _ = self._forward_fg(fg, it, "render_fg")
            bg_rgb = None
            if bg is not None:
                bws, _, _ = self._forward_bg(bg, it, head, "render_bg")
                bg_rgb = bws["bg_rgb"]
            pbg = out[1][a:b] if out[1] is not None else None
            call("psdf_nerf_loss_forward", *fg._rsp(), fws["x"], fws["density"].view(-1), fg.samples_dt.view(-1), *head, bg_rgb, None, None,
                 None, 0.0, out[0][a:b], out[2][a:b], torch.empty(b - a, 1, device=o.device), pbg, None, None, None)
        return tuple(out)

    def train(self):
        for m in self.models:
            m.train()

    def eval(self):
        for m in self.models:
            m.eval()

    # ------------------------------------------------------------------------------------ CUDA-graph replay
    def enable_cuda_graph(self):
        """later steps of the direct sequence (and the occupancy refresh) replay captured CUDA graphs: the first step of a shape runs
        eagerly, the next one is captured; re-captures follow where the captured control flow of the windows changes (iteration 1 for the
        foreground, background_nr_iters_for_c2f for the background). Containers keep their capacity and the samplers' generators live on
        the device while this is on. The autograd formulation is not captured."""
        if not self.direct:
            raise RuntimeError("NerfTrainer.enable_cuda_graph: the autograd formulation is not captured (%s)" % self.execution["step"])
        if self._cg is None:
            RaySamplesPacked.static_capacity = True
            for r in (OccupancyGrid.m_rng, RaySampler.m_rng):
                r.to_device()
            self._cg = dict(stream=torch.cuda.Stream(device=self.optimizer.flat_param.device), captures=0, graphs={}, warm={})
            self.execution["step"] = "direct kernel sequence (nerf_train.py), CUDA-graph replay"

    def disable_cuda_graph(self):
        if self._cg is not None:
            self.execution["step"] = "direct kernel sequence (nerf_train.py)"
            RaySamplesPacked.static_capacity = False
            for r in (OccupancyGrid.m_rng, RaySampler.m_rng):
                r.to_host()
            self._cg = None

    # ------------------------------------------------------------------------------------ checkpoints
    def _generators(self):
        gens = {}
        for name, r in (("occupancy", OccupancyGrid.m_rng), ("sampler", RaySampler.m_rng)):
            if r.dev is not None:
                st = r.dev.cpu().tolist()
                gens[name] = (st[0] & (2 ** 64 - 1), st[1] & (2 ** 64 - 1))
            else:
                gens[name] = (r.state, r.inc)
        gens["torch_cuda"] = torch.cuda.get_rng_state()
        return gens

    def _set_generators(self, gens):
        sg = lambda v: v - (1 << 64) if v >= (1 << 63) else v
        for name, r in (("occupancy", OccupancyGrid.m_rng), ("sampler", RaySampler.m_rng)):
            r.state, r.inc = gens[name]
            if r.dev is not None:
                r.dev.copy_(torch.tensor([sg(r.state), sg(r.inc)], dtype=torch.int64))
        torch.cuda.set_rng_state(gens["torch_cuda"].cpu())

    def save(self, ckpt_folder, experiment_name, iter_nr=None, with_optimizer=True):
        """<ckpt>/<experiment>/<iter>/models/: the five files of train_nerf.py:230-238 (nerf_hash_model.pt, nerf_hash_model_bg.pt,
        colorcal_model.pt, grid_values.pt, grid_occupancy.pt) and nerf_trainer_state.pt (optimizer moments and step count, iteration,
        generators) so that a run resumes bit for bit. -> models path"""
        it = self.iter_nr if iter_nr is None else iter_nr
        path = self.model.save(ckpt_folder, experiment_name, it)
        if self.model_bg is not None:
            self.model_bg.save(ckpt_folder, experiment_name, it, additional_name="_bg")
        if self.model_colorcal is not None:
            self.model_colorcal.save(ckpt_folder, experiment_name, it)
        torch.save(self.occupancy_grid.get_grid_values(), os.path.join(path, "grid_values.pt"))
        torch.save(self.occupancy_grid.get_grid_occupancy(), os.path.join(path, "grid_occupancy.pt"))
        if with_optimizer:
            torch.save({"optimizer": self.optimizer.state_dict(), "iter_nr": self.iter_nr, "generators": self._generators()},
                       os.path.join(path, "nerf_trainer_state.pt"))
        return path

    def load(self, ckpt_path_full, with_optimizer=True):
        """inverse of save(); a checkpoint of the reference (the five files only) loads with iter_nr = 0 and the optimizer left as it is.
        Parameters and grid are copied into the existing storages, so the flat-buffer optimizer's views and captured graphs stay valid."""
        dev = self.aabb.m_center_tensor.device
        ld = lambda f: torch.load(os.path.join(ckpt_path_full, f), map_location=dev)
        self.model.load_state_dict(ld("nerf_hash_model.pt"))
        if self.model_bg is not None:
            self.model_bg.load_state_dict(ld("nerf_hash_model_bg.pt"))
        if self.model_colorcal is not None:
            self.model_colorcal.load_state_dict(ld("colorcal_model.pt"))
        self.occupancy_grid.get_grid_values().copy_(ld("grid_values.pt"))
        self.occupancy_grid.get_grid_occupancy().copy_(ld("grid_occupancy.pt"))
        st = os.path.join(ckpt_path_full, "nerf_trainer_state.pt")
        if with_optimizer and os.path.exists(st):
            sd = torch.load(st, map_location=dev, weights_only=False)
            self.optimizer.load_state_dict(sd["optimizer"])
            self.iter_nr = int(sd["iter_nr"])
            self._set_generators(sd["generators"])
        else:
            self.iter_nr = 0
        for m in self.models:
            m.fused.pack(m.fused.params())
