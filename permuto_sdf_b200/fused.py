"""Fused evaluation of the SDF model (encoding + MLP in one tensor-core kernel, csrc/fused_sdf.cu).

`FusedSDF(model_sdf)` wraps a `models.SDF` and evaluates sdf / d sdf/dx / geometric feature without
materialising encoded features or hidden activations in HBM. It is used where no parameter gradient is
needed: SDF importance sampling, the occupancy-grid refresh, sphere tracing and normals. Training-time
evaluations that need parameter gradients go through the differentiable modules (models.SDF).
A space-time SDF (SDF(4, ...), positions (x, y, z, t)) is evaluated too; its gradient is the spatial one.
"""
import torch

from ._lib import call, load_library
from .permuto_sdf import RaySamplesPacked


def splitk_tn(a, b, slabs=64):
    """a^T b for tall operands a [R, M], b [R, K] (weight gradients: the reduction runs over the sample axis). A plain library
    GEMM gives this to one or two CTAs looping over all R rows (latency bound); as a batched GEMM over
    `slabs` row slabs followed by a small sum it fills the GPU."""
    R = a.shape[0]
    if R < 32 * slabs:
        return a.t() @ b
    main = R // slabs * slabs
    out = torch.bmm(a[:main].view(slabs, -1, a.shape[1]).transpose(1, 2), b[:main].view(slabs, -1, b.shape[1])).sum(0)
    if main != R:
        out = out + a[main:].t() @ b[main:]
    return out


class SplitKLinearFn(torch.autograd.Function):
    """F.linear(x, w, bias) whose weight gradient uses splitk_tn (the MLP layers around the fused kernels)"""

    @staticmethod
    def forward(ctx, x, w, bias):
        ctx.save_for_backward(x, w)
        return torch.addmm(bias, x, w.t())

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        g = g.contiguous()
        gx = g @ w if ctx.needs_input_grad[0] else None
        gw = splitk_tn(g, x) if ctx.needs_input_grad[1] else None
        gb = g.sum(0) if ctx.needs_input_grad[2] else None
        return gx, gw, gb


class FusedSDF:
    def __init__(self, model_sdf):
        self.model = model_sdf
        enc = model_sdf.encoding
        lin = [m for m in model_sdf.mlp_sdf if isinstance(m, torch.nn.Linear)]
        if len(lin) != 4:
            raise RuntimeError("FusedSDF supports the 4-linear-layer SDF MLP of the reference (models.py:153-161)")
        if enc.pos_dim not in (3, 4) or enc.nr_feat_per_level != 2 or not enc.concat_points or enc.nr_levels % 4 != 0:
            raise RuntimeError("FusedSDF needs pos_dim 3 or 4, 2 features per level, concat_points and nr_levels % 4 == 0")
        self.pos_dim = enc.pos_dim
        self.lin = lin
        self.in_dim = lin[0].in_features
        self.hidden = lin[0].out_features
        self.out_dim = lin[3].out_features
        if self.in_dim != enc.output_dims() or self.hidden % 16 != 0 or self.hidden > 64 or self.out_dim > 64 or self.in_dim > 64:
            raise RuntimeError("unsupported MLP shape for the fused kernel")
        lib = load_library()
        self.blob = torch.empty(int(lib.psdf_sdf_mlp_blob_bytes(self.in_dim, self.hidden, self.out_dim)), dtype=torch.uint8,
                                device=enc.lattice_values.device)
        self._versions = None
        self._pending = []              # queued backward calls of the running autograd pass (batch_backward)
        self.batch_backward = True      # with in-place gradients: one backward launch per iteration instead of one per forward call
        self.repack()

    def _cur_versions(self):
        return tuple(p._version for l in self.lin for p in (l.weight, l.bias))

    def repack(self, advance=None):
        """weights -> tensor-core operand blob (call after every optimizer step; cheap, one small kernel). advance = (step_dev, it_dev):
        the same launch also increments the device-resident AdamW step count and iteration number (either may be None)"""
        l = self.lin
        w = (l[0].weight.detach(), l[0].bias.detach(), l[1].weight.detach(), l[1].bias.detach(), l[2].weight.detach(), l[2].bias.detach(),
             l[3].weight.detach(), l[3].bias.detach())
        if advance is not None:
            call("psdf_sdf_mlp_pack_advance", self.in_dim, self.hidden, self.out_dim, *w, self.blob, advance[0], advance[1])
        else:
            call("psdf_sdf_mlp_pack", self.in_dim, self.hidden, self.out_dim, *w, self.blob)
        self._versions = self._cur_versions()

    # ------------------------------------------------------------------------------------------ training path
    def train_forward(self, points, iter_nr):
        """differentiable (wrt lattice + MLP parameters) sdf, d sdf/dx, geom in two fused kernels (forward, backward).
        Equivalent to SDF.get_sdf_and_gradient(points, iter_nr) followed by loss.backward() through its double backward;
        the gradient wrt `points` is not produced (it only matters for the 1e-4-scaled shift of the curvature loss). pos_dim 3 only: the
        space-time SDF's get_sdf_and_gradient returns the time derivative too ([N,4]), which the fused pair does not form."""
        if self.pos_dim != 3:
            raise RuntimeError("FusedSDF.train_forward: pos_dim %d; get_sdf_and_gradient of a space-time SDF returns the [N,4] gradient "
                               "including d sdf / dt, which the fused pair does not form (SpaceTimeFit runs the fused kernels directly)"
                               % self.pos_dim)
        if self._versions != self._cur_versions():
            self.repack()
        m = self.model
        m.last_iter_nr = iter_nr
        window = m.window(iter_nr).view(-1).contiguous()
        l = self.lin
        return _FusedSDFTrainFn.apply(points.detach().contiguous(), m.encoding.lattice_values, l[0].weight, l[0].bias, l[1].weight, l[1].bias,
                                      l[2].weight, l[2].bias, l[3].weight, l[3].bias, window, self)

    @torch.no_grad()
    def __call__(self, points, iter_nr, with_gradient=False, with_geom=True):
        """points [N, pos_dim] -> (sdf [N,1], gradient [N,3] or None, geom_feat [N,out-1] or None). For a space-time SDF (pos_dim 4,
        points (x, y, z, t)) the gradient is the spatial one, d sdf / d (x, y, z): the first three columns of the reference's
        get_sdf_and_gradient, all that train_4d_sdf.py reads of it."""
        if self._versions != self._cur_versions():
            self.repack()
        m, enc = self.model, self.model.encoding
        m.last_iter_nr = iter_nr
        pts = points.detach().contiguous()
        N = pts.shape[0]
        dev = pts.device
        sdf = torch.empty(N, 1, device=dev)
        grad = torch.empty(N, 3, device=dev) if with_gradient else None
        geom = torch.empty(N, self.out_dim - 1, device=dev) if (with_geom and self.out_dim > 1) else None
        window = m.window(iter_nr).view(-1).contiguous()
        fwd = ("psdf_sdf_fused_forward",) if self.pos_dim == 3 else ("psdf_sdf_fused_forward_dim", self.pos_dim)
        call(*fwd, N, enc.nr_levels, enc.capacity, pts, enc.lattice_values.detach(), enc.scale_factor,
             enc.shift_tensor(), window, enc.concat_points_scaling, self.hidden, self.out_dim, self.blob, sdf, grad, geom)
        return sdf, grad, geom


def _trace_boundary(model):
    """-> (boundary_kind, boundary[6]) of psdf_sdf_sphere_trace_dim for the model's boundary_primitive; RuntimeError for other primitives"""
    from .permuto_sdf import AABB, Sphere
    b = model.boundary_primitive
    if isinstance(b, Sphere):
        return 0, [b.m_radius] + list(b.m_center) + [0.0, 0.0]
    if isinstance(b, AABB):
        # the fp32 values check_point_inside_primitive compares against: max_bounds (s / 2 rounded once) and the translation
        return 1, [float(v) for v in b.max_bounds] + list(b.bounding_box_translation)
    raise RuntimeError("FusedSDF.sphere_trace: the model's boundary_primitive is a %s; the fused tracer tests against a Sphere or an AABB"
                       % type(b).__name__)


def _fused_sdf_sphere_trace(self, points, dirs, iter_nr, nr_iters, sdf_multiplier, sdf_converged_tresh, occupancy_grid=None, time_val=None):
    """sphere_trace's iteration loop (sdf_utils.py:150-200) in one kernel: -> (traced points [N,3], converged [N] bool).
    With an occupancy grid every step is followed by advance_sample_to_next_occupied_voxel, otherwise rays stop when they leave the
    model's boundary_primitive (a Sphere or an AABB). A space-time SDF (pos_dim 4) is traced at `time_val`: the network sees
    (x, y, z, time_val) as the reference's loop feeds it, the points and the steps stay 3-D."""
    if self.pos_dim == 4 and time_val is None:
        raise RuntimeError("FusedSDF.sphere_trace: pos_dim 4; a space-time SDF is traced at a time value (time_val=...)")
    if self.pos_dim == 3 and time_val is not None:
        raise RuntimeError("FusedSDF.sphere_trace: time_val given for a pos_dim 3 SDF, which has no time input")
    kind, boundary = _trace_boundary(self.model)
    if self._versions != self._cur_versions():
        self.repack()
    m, enc = self.model, self.model.encoding
    pts, drs = points.detach().contiguous(), dirs.detach().contiguous()
    N = pts.shape[0]
    out = torch.empty_like(pts)
    conv = torch.empty(N, dtype=torch.bool, device=pts.device)
    queue = torch.zeros(8, dtype=torch.int32, device=pts.device)        # [0] ray queue of the persistent CTAs, [1..4] statistics
    self.last_trace_stats = queue
    window = m.window(iter_nr).view(-1).contiguous()
    if occupancy_grid is not None:
        V, e, t = occupancy_grid._geom()
        occ = occupancy_grid.m_grid_occupancy
    else:
        V, e, t, occ = 1, 1.0, [0.0, 0.0, 0.0], None
    net = (N, enc.nr_levels, enc.capacity, pts, drs, enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(), window,
           enc.concat_points_scaling, self.hidden, self.out_dim, self.blob, int(nr_iters), float(sdf_multiplier), float(sdf_converged_tresh),
           occ, V, e, t)
    with torch.no_grad():
        if self.pos_dim == 3 and kind == 0:         # the original entry point: the (3, sphere) case of psdf_sdf_sphere_trace_dim
            call("psdf_sdf_sphere_trace", *net, boundary[0], boundary[1:4], out, conv, queue)
        else:
            call("psdf_sdf_sphere_trace_dim", self.pos_dim, 0.0 if time_val is None else float(time_val), kind, boundary, *net, out, conv,
                 queue)
    return out, conv


FusedSDF.sphere_trace = _fused_sdf_sphere_trace


def _pad16(v):
    return (v + 15) // 16 * 16


class _FusedSDFTrainFn(torch.autograd.Function):
    """forward: psdf_sdf_fused_forward (value + 3 tangent streams); backward: psdf_sdf_fused_backward (value + the tangent
    along the upstream gradient, reverse sweep and weight gradients on the tensor cores, then the lattice-scatter kernel)."""

    @staticmethod
    def forward(ctx, points, lattice, W0, b0, W1, b1, W2, b2, W3, b3, window, fused):
        enc = fused.model.encoding
        N = points.shape[0]
        dev = points.device
        sdf = torch.empty(N, 1, device=dev)
        grad = torch.empty(N, 3, device=dev)
        geom = torch.empty(N, fused.out_dim - 1, device=dev)
        call("psdf_sdf_fused_forward", N, enc.nr_levels, enc.capacity, points, lattice.detach(), enc.scale_factor, enc.shift_tensor(), window,
             enc.concat_points_scaling, fused.hidden, fused.out_dim, fused.blob, sdf, grad, geom)
        ctx.fused = fused
        ctx.save_for_backward(points, lattice, window)
        return sdf, grad, geom

    @staticmethod
    def backward(ctx, g_sdf, g_grad, g_geom):
        fused = ctx.fused
        points, lattice, window = ctx.saved_tensors
        enc = fused.model.encoding
        N = points.shape[0]
        dev = points.device
        dims_k = [fused.in_dim, fused.hidden, fused.hidden, fused.hidden]
        dims_n = [fused.hidden, fused.hidden, fused.hidden, fused.out_dim]
        # with a flat-buffer optimizer the gradients are accumulated straight into the persistent .grad buffers (hash table:
        # no 33 MB zero-fill plus accumulate pass per call; MLP: no zero-fills / add_ per tensor); autograd then gets no
        # gradient for those parameters from this node
        params = [p for l in fused.lin for p in (l.weight, l.bias)]
        in_place = getattr(enc, "grad_in_place", False) and lattice.grad is not None and lattice.grad.is_contiguous() and \
            all(p.grad is not None and p.grad.is_contiguous() for p in params)
        if in_place:
            gW, gb = [l.weight.grad for l in fused.lin], [l.bias.grad for l in fused.lin]
        else:
            gW = [torch.zeros(n, k, device=dev) for n, k in zip(dims_n, dims_k)]
            gb = [torch.zeros(n, device=dev) for n in dims_n]
        g_lat = lattice.grad if in_place else torch.zeros_like(lattice)
        c = lambda t: None if t is None else t.contiguous()
        if in_place and fused.batch_backward:
            # gradients accumulate in the persistent .grad buffers and autograd gets nothing back from this node, so the launch can wait:
            # every backward of this iteration (main samples, curvature pass, off-surface points) is queued and ONE kernel processes them
            # all when the autograd pass has finished (engine callback) -- see psdf_sdf_fused_backward_multi
            fused._queue_backward(points, c(g_sdf), c(g_grad), c(g_geom), window)
            return (None,) * 12
        ws = torch.empty(int(load_library().psdf_sdf_fused_backward_workspace_bytes(N)), dtype=torch.uint8, device=dev)
        call("psdf_sdf_fused_backward", N, enc.nr_levels, enc.capacity, points, lattice.detach(), enc.scale_factor, enc.shift_tensor(), window,
             enc.concat_points_scaling, fused.hidden, fused.out_dim, fused.blob, c(g_sdf), c(g_grad), c(g_geom), g_lat, ws, gW[0], gW[1], gW[2],
             gW[3], gb[0], gb[1], gb[2], gb[3])
        if in_place:
            return (None,) * 12
        return (None, g_lat, gW[0], gb[0], gW[1], gb[1], gW[2], gb[2], gW[3], gb[3], None, None)


def _fused_sdf_queue_backward(self, points, g_sdf, g_grad, g_geom, window):
    if not self._pending:
        torch.autograd.Variable._execution_engine.queue_callback(self._flush_backward)
    self._pending.append((points, g_sdf, g_grad, g_geom, window))


def _fused_sdf_flush_backward(self):
    """one launch per group of <= 3 queued sample sets that share the coarse-to-fine window"""
    pend, self._pending = self._pending, []
    enc = self.model.encoding
    lattice = enc.lattice_values
    lib = load_library()
    while pend:
        w0 = pend[0][4]
        batch = [p for p in pend if p[4].data_ptr() == w0.data_ptr()][:3]
        pend = [p for p in pend if not any(p is b for b in batch)]
        batch.sort(key=lambda p: -p[0].shape[0])
        segs = batch + [None] * (3 - len(batch))
        ns = [0 if s is None else s[0].shape[0] for s in segs]
        ws = torch.empty(int(lib.psdf_sdf_fused_backward_multi_workspace_bytes(*ns)), dtype=torch.uint8, device=lattice.device)
        flat = []
        for s, n in zip(segs, ns):
            flat += [n] + ([None] * 4 if s is None else [s[0], s[1], s[2], s[3]])
        call("psdf_sdf_fused_backward_multi", enc.nr_levels, enc.capacity, lattice.detach(), enc.scale_factor, enc.shift_tensor(), w0,
             enc.concat_points_scaling, self.hidden, self.out_dim, self.blob, *flat, lattice.grad, ws,
             self.lin[0].weight.grad, self.lin[1].weight.grad, self.lin[2].weight.grad, self.lin[3].weight.grad,
             self.lin[0].bias.grad, self.lin[1].bias.grad, self.lin[2].bias.grad, self.lin[3].bias.grad)


FusedSDF._queue_backward = _fused_sdf_queue_backward
FusedSDF._flush_backward = _fused_sdf_flush_backward


# ================================================================================================ NeuS compositing + losses
class _NeusRenderLossFn(torch.autograd.Function):
    """psdf_neus_render_loss_forward / _backward (csrc/neus_fused.cu): alpha, transmittance, weights, integration and the
    rgb / mask / eikonal loss terms of one training iteration in a single launch each way
    (volume_rendering_modules.py:129-176 + train_permuto_sdf.py:349-383)."""

    @staticmethod
    def forward(ctx, rsp, sdf, grad, rgb, inv_s, bg_rgb, cos_anneal, gt_rgb, gt_mask, hit, w_eik, w_mask):
        R = rsp.ray_start_end_idx.shape[0]
        N = sdf.shape[0]
        dev = sdf.device
        alpha = torch.empty(N, device=dev)
        T = torch.empty(N, device=dev)
        w = torch.zeros(N, 1, device=dev)
        pred = torch.empty(R, 3, device=dev)
        wsum = torch.empty(R, 1, device=dev)
        bgT = torch.empty(R, 1, device=dev)
        ray_loss = torch.empty(R, 3, device=dev)
        sdf_c, grad_c, rgb_c = sdf.detach().contiguous(), grad.detach().contiguous(), rgb.detach().contiguous()
        inv_s_c = inv_s.detach().reshape(1).contiguous()
        bg_c = None if bg_rgb is None else bg_rgb.detach().contiguous()
        # schedule values / sample count that live on the device (static-capacity containers under CUDA-graph replay)
        cos_dev = cos_anneal.detach().reshape(1).float().contiguous() if isinstance(cos_anneal, torch.Tensor) else None
        cos_f = 0.0 if cos_dev is not None else float(cos_anneal)
        n_dev = rsp.cur_nr_samples if RaySamplesPacked.static_capacity else None
        # data-parallel runs: the eikonal term is a mean over the samples of ALL ranks -> divide by the mean per-rank sample count
        # (set by train.run_net after an 8-byte all-reduce) instead of the local one, so that the rank-averaged gradient equals the
        # gradient of the global batch (SURVEY.md 8e)
        n_dev = getattr(rsp, "dp_mean_nr_samples", None) if getattr(rsp, "dp_mean_nr_samples", None) is not None else n_dev
        call("psdf_neus_render_loss_forward", *rsp._rsp(), sdf_c, grad_c, rgb_c, rsp.samples_dirs, rsp.samples_dt, inv_s_c, cos_f, cos_dev,
             gt_rgb, gt_mask, hit, bg_c, alpha, T, w, pred, wsum, bgT, ray_loss)
        terms = ray_loss.sum(0)
        c_rgb, c_mask = 1.0 / (3 * R), (w_mask / R) if gt_mask is not None else 0.0
        if n_dev is None:
            c_eik = w_eik / max(N, 1)
            loss = terms[0] * c_rgb + terms[1] * c_mask + terms[2] * c_eik
        else:
            c_eik = w_eik           # divided by the device-side sample count
            loss = terms[0] * c_rgb + terms[1] * c_mask + terms[2] * (w_eik / n_dev.clamp(min=1).float()).squeeze(0)
        ctx.rsp = rsp
        ctx.cfg = (cos_f, cos_dev, gt_rgb, gt_mask, hit, c_rgb, c_mask, c_eik, n_dev)
        ctx.has_bg = bg_rgb is not None
        ctx.save_for_backward(sdf_c, grad_c, rgb_c, inv_s_c, bg_c, alpha, T, pred, wsum, bgT)
        ctx.mark_non_differentiable(pred, wsum, w, terms)
        return loss, pred, wsum, w, terms

    @staticmethod
    def backward(ctx, g_loss, *_):
        sdf, grad, rgb, inv_s, bg, alpha, T, pred, wsum, bgT = ctx.saved_tensors
        rsp = ctx.rsp
        cos_f, cos_dev, gt_rgb, gt_mask, hit, s_rgb, s_mask, s_eik, n_dev = ctx.cfg
        # rows outside every ray (gaps of slot-strided containers, the zero tail of static-capacity ones) get no gradient
        flat = torch.zeros(sdf.shape[0] * 7, device=sdf.device)            # one zero-fill for the three gradients
        n1 = sdf.shape[0]
        g_sdf, g_grad, g_rgb = flat[:n1].view_as(sdf), flat[n1:4 * n1].view_as(grad), flat[4 * n1:].view_as(rgb)
        g_bg = torch.empty_like(bg) if ctx.has_bg and ctx.needs_input_grad[5] else None
        g_inv = torch.zeros(1, device=sdf.device) if ctx.needs_input_grad[4] else None
        call("psdf_neus_render_loss_backward", *rsp._rsp(), sdf, grad, rgb, rsp.samples_dirs, rsp.samples_dt, inv_s, cos_f, cos_dev, gt_rgb,
             gt_mask, hit, bg, alpha, T, pred, wsum, bgT, g_loss.reshape(1).contiguous(), s_rgb, s_mask, s_eik, n_dev, g_sdf, g_grad, g_rgb,
             g_bg, g_inv)
        ctx.rsp = None
        return (None, g_sdf, g_grad, g_rgb, None if g_inv is None else g_inv.reshape(()), g_bg, None, None, None, None, None, None)


def neus_render_loss(rsp, sdf, sdf_gradients, rgb_samples, inv_s, cos_anneal_ratio, gt_rgb, gt_mask, hit, eikonal_weight, mask_weight,
                     bg_rgb=None):
    """-> (loss = rgb L1 + eikonal_weight * eikonal + mask_weight * BCE, pred_rgb [R,3], weights_sum [R,1], weights [N,1],
    terms [3] = per-term sums). `inv_s` is the un-clipped 0-d tensor of SingleVarianceNetwork; `hit` bool/u8 [R] or None."""
    load_library()
    f = lambda t: None if t is None else t.detach().reshape(-1).contiguous().float()
    hit_u8 = None if hit is None else hit.detach().reshape(-1).to(torch.uint8)
    if sdf.shape[0] != rsp.samples_dirs.shape[0]:
        raise ValueError("neus_render_loss: sdf must have one row per packed sample")
    return _NeusRenderLossFn.apply(rsp, sdf.reshape(-1), sdf_gradients, rgb_samples, inv_s, bg_rgb, cos_anneal_ratio,
                                   gt_rgb.detach().contiguous(), f(gt_mask), hit_u8, float(eikonal_weight), float(mask_weight))


# ================================================================================================ colour-network helpers
class LipschitzNormFn(torch.autograd.Function):
    """LipshitzMLP.normalization (models.py:96-110) in one kernel each way (csrc/rgb_misc.cu): w * min(1, softplus(c) / sum|w|)"""

    @staticmethod
    def forward(ctx, w, c):
        wc, cc = w.detach().contiguous(), c.detach().reshape(1).contiguous()
        out = torch.empty_like(wc)
        call("psdf_lipschitz_normalize", wc.shape[0], wc.shape[1], wc, cc, out)
        ctx.save_for_backward(wc, cc)
        return out

    @staticmethod
    def backward(ctx, g):
        wc, cc = ctx.saved_tensors
        gw = torch.empty_like(wc)
        gc = torch.zeros(1, device=wc.device) if ctx.needs_input_grad[1] else None
        call("psdf_lipschitz_normalize_backward", wc.shape[0], wc.shape[1], wc, cc, g.contiguous(), gw, gc)
        return gw, gc


class CalibSigmoidFn(torch.autograd.Function):
    """Colorcal.calib_RGB_samples_packed followed by the sigmoid of the colour head (models.py:395-414, 677-741) on packed samples,
    one kernel each way; img_indices is per ray; rows outside every ray stay zero"""

    @staticmethod
    def forward(ctx, x, ray_start_end_idx, img_indices, weight_delta, bias, fixed_img):
        xc = x.detach().contiguous()
        out = torch.zeros_like(xc)
        R, N = ray_start_end_idx.shape[0], xc.shape[0]
        img = None if img_indices is None else img_indices.detach().reshape(-1).to(torch.int32).contiguous()
        wd = None if weight_delta is None else weight_delta.detach().contiguous()
        bs = None if bias is None else bias.detach().contiguous()
        rsp = (R, N, ray_start_end_idx, 0, 0)
        call("psdf_calib_sigmoid_forward", *rsp, xc, img if wd is not None else None, wd, bs, int(fixed_img), out)
        ctx.rsp, ctx.fixed = rsp, int(fixed_img)
        ctx.save_for_backward(xc, out, img, wd)
        return out

    @staticmethod
    def backward(ctx, g):
        xc, out, img, wd = ctx.saved_tensors
        gx = torch.zeros_like(xc)
        need_p = wd is not None and (ctx.needs_input_grad[3] or ctx.needs_input_grad[4])
        gwd = torch.zeros_like(wd) if need_p else None
        gbs = torch.zeros_like(wd) if need_p else None
        call("psdf_calib_sigmoid_backward", *ctx.rsp, xc, out, g.contiguous(), img if wd is not None else None, wd, ctx.fixed, gx, gwd, gbs)
        return gx, None, None, gwd, gbs, None


# ================================================================================================ fused colour network
class FusedRGB:
    """models.RGB on the tensor cores (csrc/fused_rgb.cu, fused_rgb_bwd.cu): encoding + SH + normal + geom -> Lipschitz MLP.
    The Lipschitz normalisation of the weights stays a (differentiable) per-layer kernel outside; the fused kernels see the
    normalised matrices W_eff through a packed operand blob."""

    def __init__(self, model_rgb):
        self.model = model_rgb
        enc = model_rgb.encoding
        self.layers = list(model_rgb.mlp.layers)
        if len(self.layers) != 4 or self.layers[3].out_features != 3 or not model_rgb.mlp.last_layer_linear:
            raise RuntimeError("FusedRGB supports the 4-layer colour MLP of the reference (models.py:330-340)")
        if enc.pos_dim != 3 or enc.nr_feat_per_level != 2 or not enc.concat_points or enc.nr_levels % 4 != 0:
            raise RuntimeError("FusedRGB needs pos_dim 3, 2 features per level, concat_points and nr_levels % 4 == 0")
        self.in_dim = self.layers[0].in_features
        self.h = [l.out_features for l in self.layers[:3]]
        if self.in_dim != enc.output_dims() + 25 + 3 + 32 or self.in_dim > 128 or any(h > 128 or h % 16 for h in self.h):
            raise RuntimeError("unsupported colour MLP shape for the fused kernel")
        lib = load_library()
        self.blob = torch.empty(int(lib.psdf_rgb_mlp_blob_bytes(self.in_dim, *self.h, 3)), dtype=torch.uint8, device=enc.lattice_values.device)

    def normalized_weights(self):
        mlp = self.model.mlp
        return [LipschitzNormFn.apply(l.weight, mlp.lipshitz_bound_per_layer[i]) for i, l in enumerate(self.layers)]

    def pack(self, w_eff):
        l = self.layers
        call("psdf_rgb_mlp_pack", self.in_dim, *self.h, 3, w_eff[0].detach(), l[0].bias.detach(), w_eff[1].detach(), l[1].bias.detach(),
             w_eff[2].detach(), l[2].bias.detach(), w_eff[3].detach(), l[3].bias.detach(), self.blob)

    def _window(self, iter_nr):
        from .models import map_range_val
        m = self.model
        m.last_iter_nr = int(iter_nr)
        return m.c2f(map_range_val(iter_nr, 0.0, m.nr_iters_for_c2f, 0.3, 1.0)).view(-1).contiguous()

    @torch.no_grad()
    def __call__(self, points, samples_dirs, sdf_gradients, geom_feat, iter_nr):
        """-> linear colour [N,3] (before calibration / sigmoid), no autograd"""
        self.pack(self.normalized_weights())
        enc = self.model.encoding
        N = points.shape[0]
        out = torch.empty(N, 3, device=points.device)
        call("psdf_rgb_fused_forward", N, enc.nr_levels, enc.capacity, points.contiguous(), samples_dirs.contiguous(),
             sdf_gradients.contiguous(), geom_feat.contiguous(), geom_feat.shape[1], enc.lattice_values.detach(), enc.scale_factor,
             enc.shift_tensor(), self._window(iter_nr), enc.concat_points_scaling, *self.h, self.blob, out)
        return out


class _FusedRGBTrainFn(torch.autograd.Function):
    """forward: psdf_rgb_fused_forward; backward: psdf_rgb_fused_backward (reverse sweep + tensor-core dW). Differentiable wrt the
    hash table, the (normalised) weights, the biases, the sdf gradients and the geometric feature; not wrt points / view dirs."""

    @staticmethod
    def forward(ctx, points, dirs, sdf_grad, geom, lattice, w0, b0, w1, b1, w2, b2, w3, b3, window, fr):
        enc = fr.model.encoding
        fr.pack([w0, w1, w2, w3])
        N = points.shape[0]
        out = torch.empty(N, 3, device=points.device)
        sg, gm = sdf_grad.detach().contiguous(), geom.detach().contiguous()
        call("psdf_rgb_fused_forward", N, enc.nr_levels, enc.capacity, points, dirs, sg, gm, gm.shape[1], lattice.detach(), enc.scale_factor,
             enc.shift_tensor(), window, enc.concat_points_scaling, *fr.h, fr.blob, out)
        ctx.fr = fr
        ctx.save_for_backward(points, dirs, sg, gm, lattice, window)
        return out

    @staticmethod
    def backward(ctx, g_out):
        fr = ctx.fr
        points, dirs, sg, gm, lattice, window = ctx.saved_tensors
        enc = fr.model.encoding
        N = points.shape[0]
        dev = points.device
        dims = [fr.in_dim] + fr.h + [3]
        in_place = getattr(enc, "grad_in_place", False) and lattice.grad is not None and lattice.grad.is_contiguous() and \
            all(l.bias.grad is not None and l.bias.grad.is_contiguous() for l in fr.layers)
        sizes = [dims[l + 1] * dims[l] for l in range(4)]                           # wrt the normalised weights: flows on through autograd
        offs = [0, sizes[0], sizes[0] + sizes[1], sizes[0] + sizes[1] + sizes[2]]
        flat_w = torch.zeros(sum(sizes), device=dev)                                # one zero-fill for the four matrices
        gW = [flat_w[offs[l]:offs[l] + sizes[l]].view(dims[l + 1], dims[l]) for l in range(4)]
        gb = [l.bias.grad for l in fr.layers] if in_place else [torch.zeros(dims[l + 1], device=dev) for l in range(4)]
        g_sg = torch.empty_like(sg)          # every row is written by the kernel
        g_gm = torch.empty_like(gm)
        ws = torch.empty(int(load_library().psdf_rgb_fused_backward_workspace_bytes(N)), dtype=torch.uint8, device=dev)
        g_lat = lattice.grad if in_place else torch.zeros_like(lattice)
        # the packed blob still holds this iteration's weights (pack happens in forward, one forward per iteration)
        call("psdf_rgb_fused_backward", N, enc.nr_levels, enc.capacity, points, dirs, sg, gm, gm.shape[1], lattice.detach(), enc.scale_factor,
             enc.shift_tensor(), window, enc.concat_points_scaling, *fr.h, fr.blob, g_out.contiguous(), g_lat, g_sg, g_gm, ws, gW[0], gW[1],
             gW[2], gW[3], gb[0], gb[1], gb[2], gb[3])
        if in_place and getattr(fr, "after_backward", None) is not None:
            fr.after_backward()          # data-parallel: the colour hash-table gradient is final -> its all-reduce starts now
        if in_place:
            return (None, None, g_sg, g_gm, None, gW[0], None, gW[1], None, gW[2], None, gW[3], None, None, None)
        return (None, None, g_sg, g_gm, g_lat, gW[0], gb[0], gW[1], gb[1], gW[2], gb[2], gW[3], gb[3], None, None)


def _fused_rgb_train_forward(self, points, samples_dirs, sdf_gradients, geom_feat, iter_nr):
    """differentiable linear colour [N,3]: Lipschitz normalisation (kernel pair per layer) -> fused forward / backward"""
    w = self.normalized_weights()
    l = self.layers
    return _FusedRGBTrainFn.apply(points.detach().contiguous(), samples_dirs.detach().contiguous(), sdf_gradients, geom_feat,
                                  self.model.encoding.lattice_values, w[0], l[0].bias, w[1], l[1].bias, w[2], l[2].bias, w[3], l[3].bias,
                                  self._window(iter_nr), self)


FusedRGB.train_forward = _fused_rgb_train_forward


# ================================================================================================ fused background network
class FusedNerfHash:
    """models.NerfHash on the tensor cores (csrc/fused_bg.cu): 3-D (foreground NeRF) or 4-D (NeRF++ background) encoding -> trunk
    (density) -> colour head, seven layers in one kernel each way. Produces the linear colour (before calibration / sigmoid) and the
    density."""

    def __init__(self, model_bg):
        self.model = model_bg
        enc = model_bg.encoding
        trunk = [m for m in model_bg.mlp_feat_and_density if isinstance(m, torch.nn.Linear)]
        head = [m for m in model_bg.mlp_rgb if isinstance(m, torch.nn.Linear)]
        self.lin = trunk + head
        dims = [(l.in_features, l.out_features) for l in self.lin]
        if enc.pos_dim not in (3, 4) or enc.nr_feat_per_level != 2 or not enc.concat_points or enc.nr_levels % 4 != 0:
            raise RuntimeError("FusedNerfHash needs pos_dim 3 or 4, 2 features per level, concat_points and nr_levels % 4 == 0")
        self.pos_dim = enc.pos_dim
        self.in_dim = enc.output_dims()
        want = [(self.in_dim, 64), (64, 64), (64, 64), (64, 65), (80, 64), (64, 64), (64, 3)]
        if dims != want:
            raise RuntimeError("FusedNerfHash supports the 7-layer NerfHash MLPs of the reference (models.py:437-447), got %s" % dims)
        lib = load_library()
        nbytes = int(lib.psdf_bg_mlp_blob_bytes(self.in_dim))
        if nbytes == 0:
            raise RuntimeError("FusedNerfHash: %d encoder columns are more than the fused kernel takes (nr_levels <= 28)" % self.in_dim)
        self.blob = torch.empty(nbytes, dtype=torch.uint8, device=enc.lattice_values.device)

    def params(self):
        return [p for l in self.lin for p in (l.weight, l.bias)]

    def pack(self, params):
        call("psdf_bg_mlp_pack", self.in_dim, *[p.detach() for p in params], self.blob)
        self.packed_versions = tuple(p._version for p in params)

    def _window(self, iter_nr, record=True):
        from .models import map_range_val
        m = self.model
        if record:
            m.last_iter_nr = int(iter_nr)
        return m.c2f(map_range_val(iter_nr, 0.0, m.nr_iters_for_c2f, 0.3, 1.0)).view(-1).contiguous()

    def _forward(self, pos, dirs, lattice, window):
        enc = self.model.encoding
        N = pos.shape[0]
        rgb = torch.empty(N, 3, device=pos.device)
        density = torch.empty(N, 1, device=pos.device)
        call("psdf_nerf_fused_forward", self.pos_dim, N, enc.nr_levels, enc.capacity, pos, dirs, lattice.detach(), enc.scale_factor,
             enc.shift_tensor(), window, enc.concat_points_scaling, self.blob, rgb, density)
        return rgb, density

    @torch.no_grad()
    def __call__(self, samples_pos, samples_dirs, iter_nr):
        """-> (linear colour [N,3], density [N,1]), no autograd"""
        self.pack(self.params())
        return self._forward(samples_pos.detach().contiguous(), samples_dirs.detach().contiguous(), self.model.encoding.lattice_values,
                             self._window(iter_nr))

    @torch.no_grad()
    def density(self, pos, iter_nr):
        """NerfHash.get_only_density (models.py:528-550) of a foreground NerfHash(3): density [N,1] at pos [N,3], no autograd, from the
        density-only kernel (encoder and trunk; the colour head is not run). Bit-identical to the density of __call__. Leaves
        model.last_iter_nr as it is, as the reference's get_only_density does."""
        if self.pos_dim != 3:
            raise RuntimeError("FusedNerfHash.density: the density-only kernel serves the 3-D NerfHash (pos_dim 3), got pos_dim %d"
                               % self.pos_dim)
        self.pack(self.params())
        enc = self.model.encoding
        pos = pos.detach().contiguous()
        density = torch.empty(pos.shape[0], 1, device=pos.device)
        call("psdf_nerf_density_forward", pos.shape[0], enc.nr_levels, enc.capacity, pos, enc.lattice_values.detach(), enc.scale_factor,
             enc.shift_tensor(), self._window(iter_nr, record=False), enc.concat_points_scaling, self.blob, density)
        return density

    def train_forward(self, samples_pos, samples_dirs, iter_nr):
        """differentiable (wrt the hash table, weights and biases) linear colour [N,3] and density [N,1]"""
        return _FusedNerfHashFn.apply(samples_pos.detach().contiguous(), samples_dirs.detach().contiguous(), self.model.encoding.lattice_values,
                                      self._window(iter_nr), self, *self.params())


class _FusedNerfHashFn(torch.autograd.Function):
    """forward: psdf_nerf_fused_forward; backward: psdf_nerf_fused_backward (reverse sweep + tensor-core dW, then the lattice scatter)"""

    @staticmethod
    def forward(ctx, pos, dirs, lattice, window, fb, *params):
        fb.pack(params)
        ctx.fb, ctx.versions = fb, fb.packed_versions
        ctx.save_for_backward(pos, dirs, lattice, window)
        return fb._forward(pos, dirs, lattice, window)

    @staticmethod
    def backward(ctx, g_rgb, g_density):
        fb = ctx.fb
        pos, dirs, lattice, window = ctx.saved_tensors
        enc = fb.model.encoding
        N = pos.shape[0]
        dev = pos.device
        params = fb.params()
        # with a flat-buffer optimizer the gradients accumulate straight into the persistent .grad buffers (as in the colour network)
        in_place = getattr(enc, "grad_in_place", False) and lattice.grad is not None and lattice.grad.is_contiguous() and \
            all(p.grad is not None and p.grad.is_contiguous() for p in params)
        grads = [p.grad for p in params] if in_place else [torch.zeros_like(p) for p in params]
        g_lat = lattice.grad if in_place else torch.zeros_like(lattice)
        g_rgb = torch.zeros(N, 3, device=dev) if g_rgb is None else g_rgb.contiguous()
        g_density = torch.zeros(N, 1, device=dev) if g_density is None else g_density.contiguous()
        ws = torch.empty(int(load_library().psdf_bg_fused_backward_workspace_bytes(N)), dtype=torch.uint8, device=dev)
        # the backward needs the weights of its forward: unchanged parameters, and the blob packed from them
        if tuple(p._version for p in params) != ctx.versions:
            raise RuntimeError("FusedNerfHash: a parameter was modified in place between the forward and its backward")
        if fb.packed_versions != ctx.versions:
            fb.pack(params)
        call("psdf_nerf_fused_backward", fb.pos_dim, N, enc.nr_levels, enc.capacity, pos, dirs, lattice.detach(), enc.scale_factor,
             enc.shift_tensor(), window, enc.concat_points_scaling, fb.blob, g_rgb, g_density, g_lat, ws, *grads[0::2], *grads[1::2])
        if in_place:
            return (None,) * (5 + len(params))
        return (None, None, g_lat, None, None) + tuple(grads)


# ================================================================================================ curvature loss
class CurvatureLossFn(torch.autograd.Function):
    """mean over the valid samples of acos(clamp(normalize(g) . normalize(g_shifted))) / pi (models.py:283-294 +
    train_permuto_sdf.py:362-366), one kernel each way (csrc/rgb_misc.cu). n_dev: device int32 [1] count of valid rows
    (static-capacity containers) or None (all rows)."""

    @staticmethod
    def forward(ctx, g, gs, n_dev):
        gc, gsc = g.detach().contiguous(), gs.detach().contiguous()
        N = gc.shape[0]
        curv = torch.empty(N, device=gc.device)
        total = torch.zeros(1, device=gc.device)
        call("psdf_curvature_loss_forward", N, gc, gsc, n_dev, curv, total)
        ctx.save_for_backward(gc, gsc, n_dev)
        ctx.N = N
        loss = total / (float(max(N, 1)) if n_dev is None else n_dev.clamp(min=1).float())
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g_loss):
        gc, gsc, n_dev = ctx.saved_tensors
        gg, ggs = torch.empty_like(gc), torch.empty_like(gsc)
        call("psdf_curvature_loss_backward", ctx.N, gc, gsc, n_dev, g_loss.reshape(1).contiguous(), 1.0 if n_dev is not None else 1.0 / max(ctx.N, 1),
             gg, ggs)
        return gg, ggs, None


def curvature_shifted_points(points, sdf_gradients, epsilon=1e-4, rnd=None):
    """points + eps * cross(normalize(sdf_gradients), normalize(randn)) (models.py:266-273), no autograd (the shifted points only feed
    a forward whose position gradient is not propagated)"""
    rnd = torch.randn_like(points) if rnd is None else rnd.contiguous()
    out = torch.empty_like(points)
    call("psdf_curvature_shift_points", points.shape[0], points.detach().contiguous(), sdf_gradients.detach().contiguous(), rnd, float(epsilon), out)
    return out
