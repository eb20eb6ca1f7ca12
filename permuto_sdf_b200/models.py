"""Hot-path models: SDF, RGB (Lipschitz MLP), background NeRF and colour calibration.

Mirror of permuto_sdf_py/models/models.py (SDF :131-307, LipshitzMLP :54-129, RGB :309-420,
NerfHash :425-563, Colorcal :677-741) on top of `permutohedral_encoding` / `permuto_sdf` of this
package. The reference hard-codes 24 levels / 32-wide SDF MLP; BASELINE.json's synthetic config wants
16 levels / 64-wide, so the sizes are constructor parameters with the reference's values as defaults
(SURVEY.md F6). Weight init follows leaky_relu_init (permuto_sdf_py/utils/common_utils.py:248-293).
"""
import math
import sys

import numpy as np
import torch
import torch.nn.functional as F

from . import permutohedral_encoding as permuto_enc
from .permuto_sdf import PermutoSDF, RaySamplesPacked
from .volume_rendering import VolumeRenderingNerf, VolumeRenderingNeus


class _LazySplitK:
    """fused.py imports models lazily; resolve SplitKLinearFn on first use"""
    fn = None

    @staticmethod
    def apply(x, w, b):
        if _LazySplitK.fn is None:
            from .fused import SplitKLinearFn as f
            _LazySplitK.fn = f
        return _LazySplitK.fn.apply(x, w, b)


SplitKLinearFn = _LazySplitK


class DeviceIter:
    """Iteration number held twice: `host` (int) drives Python control flow, `dev` (0-d float32 CUDA tensor with the same
    value) feeds every quantity that changes from one iteration to the next (map_range_val ramps). A training iteration
    captured in a CUDA graph with a DeviceIter stays valid while lo <= iteration < hi: every comparison against the
    iteration narrows [lo, hi) to the range over which the branch that was taken does not change."""

    def __init__(self, host, dev):
        self.host, self.dev = int(host), dev
        self.lo, self.hi = float("-inf"), float("inf")

    def __int__(self):
        return self.host

    __index__ = __int__

    def __float__(self):
        return float(self.host)

    def _at_least(self, bound):
        if self.host >= bound:
            self.lo = max(self.lo, bound)
            return True
        self.hi = min(self.hi, bound)
        return False

    def __ge__(self, o):
        return self._at_least(math.ceil(o))

    def __lt__(self, o):
        return not self._at_least(math.ceil(o))

    def __gt__(self, o):
        return self._at_least(math.floor(o) + 1)

    def __le__(self, o):
        return not self._at_least(math.floor(o) + 1)

    def __eq__(self, o):
        raise TypeError("DeviceIter: equality tests are not replayable; compare with <, <=, >, >=")

    __hash__ = None


def map_range_val(input_val, input_start, input_end, output_start, output_end):
    """common_utils.py:156-160 (clamps its input). For a DeviceIter the plateaus return Python floats (and narrow its validity
    range), the ramp returns a 0-d device tensor computed from the device-resident iteration."""
    if isinstance(input_val, DeviceIter):
        if input_val <= input_start:
            return output_start
        if input_val >= input_end:
            return output_end
        x = torch.clamp(input_val.dev, input_start, input_end)
        return output_start + ((output_end - output_start) / (input_end - input_start)) * (x - input_start)
    c = max(input_start, min(input_end, input_val))
    return output_start + ((output_end - output_start) / (input_end - input_start)) * (c - input_start)


def leaky_relu_init(m, negative_slope=0.2):
    if not isinstance(m, torch.nn.Linear):
        return
    gain = np.sqrt(2.0 / (1.0 + negative_slope ** 2))
    std = gain * np.sqrt(2.0 / (m.in_features + m.out_features))
    with torch.no_grad():
        m.weight.uniform_(-std * np.sqrt(3.0), std * np.sqrt(3.0))
        if m.bias is not None:
            m.bias.zero_()


def _init_stack(layers, last_linear_slope1=True):
    lin = [l for l in layers if isinstance(l, torch.nn.Linear)]
    for l in lin:
        leaky_relu_init(l, negative_slope=0.0)
    if last_linear_slope1:
        leaky_relu_init(lin[-1], negative_slope=1.0)


def make_encoding(pos_dim, nr_levels, capacity, concat_points_scaling, nr_feat_per_level=2, coarsest_scale=1.0, finest_scale=0.0001):
    scale_list = np.geomspace(coarsest_scale, finest_scale, num=nr_levels)
    return permuto_enc.PermutoEncoding(pos_dim, capacity, nr_levels, nr_feat_per_level, scale_list, appply_random_shift_per_level=True,
                                       concat_points=True, concat_points_scaling=concat_points_scaling)


class LipshitzMLP(torch.nn.Module):
    """models.py:54-129: per-layer weight rows scaled by min(1, softplus(c)/sum|w|)"""

    def __init__(self, in_channels, nr_out_channels_per_layer, last_layer_linear):
        super().__init__()
        self.last_layer_linear = last_layer_linear
        self.layers = torch.nn.ModuleList()
        for c in nr_out_channels_per_layer:
            self.layers.append(torch.nn.Linear(in_channels, c))
            in_channels = c
        for l in self.layers:
            leaky_relu_init(l, negative_slope=0.0)
        if last_layer_linear:
            leaky_relu_init(self.layers[-1], negative_slope=1.0)
        # the reference registers every weight / bias a second time (models.py:75-79), so its checkpoints carry the keys
        # mlp.weights_per_layer.N / mlp.biases_per_layer.N next to mlp.layers.N.*; same Parameter objects, same keys here
        self.weights_per_layer = torch.nn.ParameterList([l.weight for l in self.layers])
        self.biases_per_layer = torch.nn.ParameterList([l.bias for l in self.layers])
        self.lipshitz_bound_per_layer = torch.nn.ParameterList()
        for l in self.layers:
            max_w = torch.max(torch.sum(torch.abs(l.weight), dim=1))
            self.lipshitz_bound_per_layer.append(torch.nn.Parameter(torch.ones(1, device=l.weight.device) * max_w.detach() * 2))

    fused_normalization = True      # CUDA weights: one kernel each way (csrc/rgb_misc.cu) instead of ~6 + ~10 element-wise launches

    @staticmethod
    def normalization(w, softplus_ci):
        absrowsum = torch.sum(torch.abs(w), dim=1)
        scale = torch.clamp(softplus_ci / absrowsum, max=1.0)
        return w * scale[:, None]

    def lipshitz_bound_full(self):
        b = 1
        for c in self.lipshitz_bound_per_layer:
            b = b * F.softplus(c)
        return b

    def forward(self, x):
        n = len(self.layers)
        for i, l in enumerate(self.layers):
            if self.fused_normalization and l.weight.is_cuda:
                from .fused import LipschitzNormFn
                w = LipschitzNormFn.apply(l.weight, self.lipshitz_bound_per_layer[i])
            else:
                w = self.normalization(l.weight, F.softplus(self.lipshitz_bound_per_layer[i]))
            x = SplitKLinearFn.apply(x, w, l.bias) if (x.is_cuda and x.dim() == 2) else F.linear(x, w, l.bias)
            if not (i == n - 1 and self.last_layer_linear):
                x = F.gelu(x)
        return x


class _Checkpointed:
    """save() of the reference models (models.py:296-307, 393-404, 553-563, 731-741): <ckpt>/<experiment>/<iter>/models/<file>"""
    checkpoint_file = "model.pt"

    def path_to_save_model(self, ckpt_folder, experiment_name, iter_nr):
        import os
        return os.path.join(ckpt_folder, experiment_name, str(iter_nr), "models")

    def save(self, ckpt_folder, experiment_name, iter_nr, additional_name=None):
        import os
        models_path = self.path_to_save_model(ckpt_folder, experiment_name, iter_nr)
        os.makedirs(models_path, exist_ok=True)
        name = self.checkpoint_file
        if additional_name:
            stem, ext = os.path.splitext(name)
            name = stem + str(additional_name) + ext
        torch.save(self.state_dict(), os.path.join(models_path, name))
        return models_path


class SDF(torch.nn.Module, _Checkpointed):
    """models.py:131-307"""
    checkpoint_file = "sdf_model.pt"

    def __init__(self, in_channels, boundary_primitive, geom_feat_size_out, nr_iters_for_c2f, nr_levels=24, capacity=2 ** 18,
                 hidden=32, nr_hidden_layers=3):
        super().__init__()
        self.in_channels = in_channels
        self.boundary_primitive = boundary_primitive
        self.geom_feat_size_out = geom_feat_size_out
        self.encoding = make_encoding(in_channels, nr_levels, capacity, 1e-3)
        self.sdf_shift = 1e-2
        layers = [torch.nn.Linear(self.encoding.output_dims(), hidden), torch.nn.GELU()]
        for _ in range(nr_hidden_layers - 1):
            layers += [torch.nn.Linear(hidden, hidden), torch.nn.GELU()]
        layers += [torch.nn.Linear(hidden, 1 + geom_feat_size_out)]
        self.mlp_sdf = torch.nn.Sequential(*layers)
        _init_stack(self.mlp_sdf)
        with torch.no_grad():
            self.mlp_sdf[-1].bias += self.sdf_shift
        self.c2f = permuto_enc.Coarse2Fine(nr_levels)
        self.nr_iters_for_c2f = nr_iters_for_c2f
        self.last_iter_nr = sys.maxsize

    def window(self, iter_nr):
        return self.c2f(map_range_val(iter_nr, 0.0, self.nr_iters_for_c2f, 0.3, 1.0))

    def enable_fused_inference(self):
        """route gradient-free evaluations (importance sampling, occupancy refresh, sphere tracing) through the fused
        encoding+MLP tensor-core kernel (csrc/fused_sdf.cu); differentiable calls keep using the modular path"""
        from .fused import FusedSDF
        self.fused = FusedSDF(self)
        return self.fused

    def enable_fused_training(self, flag=True):
        """get_sdf_and_gradient (autograd mode) through the fused forward/backward kernels. Not for a space-time SDF (in_channels 4):
        its get_sdf_and_gradient returns d sdf / d (x, y, z, t), and the fused pair forms the spatial derivatives only; the per-op
        autograd path keeps serving it (SpaceTimeFit runs the fused kernels directly)."""
        D = self.encoding.pos_dim
        if flag and D != 3:
            raise RuntimeError("SDF.enable_fused_training: in_channels %d; get_sdf_and_gradient returns the [N,%d] gradient including "
                               "d sdf / dt, which the fused kernels do not form (they give d sdf / d(x, y, z) only)" % (D, D))
        if getattr(self, "fused", None) is None:
            self.enable_fused_inference()
        self.fused_training = bool(flag)

    def forward(self, points, iter_nr):
        assert points.shape[1] == self.in_channels, "points should be N x in_channels"
        self.last_iter_nr = int(iter_nr)
        if getattr(self, "fused", None) is not None and not torch.is_grad_enabled():
            sdf, _, geom = self.fused(points, iter_nr, with_gradient=False, with_geom=self.geom_feat_size_out != 0)
            return sdf, geom
        if getattr(self, "fused_training", False) and not points.requires_grad:
            # parameter gradients wanted, position gradient not: the fused training pair (its extra tangent streams are unused)
            sdf, _, geom = self.fused.train_forward(points, iter_nr)
            return sdf, (geom if self.geom_feat_size_out != 0 else None)
        feat = self.encoding(points, self.window(iter_nr).view(-1))
        y = self.mlp_sdf(feat)
        if self.geom_feat_size_out != 0:
            return y[:, 0:1], y[:, -self.geom_feat_size_out:]
        return y, None

    def get_sdf_and_gradient(self, points, iter_nr, method="autograd"):
        if method == "finite_difference":
            with torch.no_grad():
                eps = 1e-4
                pts = [points]
                for k in range(3):
                    p = points.clone(); p[:, k] += eps; pts.append(p)
                full = torch.cat(pts, 0)
            sdf_full, feat_full = self.forward(full, iter_nr)
            geom = feat_full.chunk(4, dim=0)[0] if feat_full is not None else None
            s = sdf_full.chunk(4, dim=0)
            grads = torch.cat([(s[1] - s[0]) / eps, (s[2] - s[0]) / eps, (s[3] - s[0]) / eps], 1)
            return s[0], grads, geom
        if getattr(self, "fused_training", False) and getattr(self, "fused", None) is not None and torch.is_grad_enabled():
            # one fused forward kernel (+ one fused backward kernel when loss.backward() runs), csrc/fused_sdf*.cu
            return self.fused.train_forward(points, iter_nr)
        with torch.set_grad_enabled(True):
            points.requires_grad_(True)
            sdf, geom = self.forward(points, iter_nr)
            grads = torch.autograd.grad(outputs=sdf, inputs=points, grad_outputs=torch.ones_like(sdf, requires_grad=False),
                                        create_graph=True, retain_graph=True, only_inputs=True)[0]
        return sdf, grads, geom

    def get_sdf_and_curvature_1d_precomputed_gradient_normal_based(self, points, sdf_gradients, iter_nr):
        """models.py:261-294"""
        epsilon = 1e-4
        rand_directions = F.normalize(torch.randn_like(points), dim=-1)
        normals = F.normalize(sdf_gradients, dim=-1)
        tangent = torch.cross(normals, rand_directions, dim=-1)
        points_shifted = points.clone() + tangent * epsilon
        sdf_shifted, grads_shifted, _ = self.get_sdf_and_gradient(points_shifted, iter_nr)
        normals_shifted = F.normalize(grads_shifted, dim=-1)
        dot = (normals * normals_shifted).sum(dim=-1, keepdim=True)
        angle = torch.acos(torch.clamp(dot, -1.0 + 1e-6, 1.0 - 1e-6))
        return sdf_shifted, angle / math.pi


    def curvature_loss(self, points, sdf_gradients, iter_nr, nr_valid_dev=None, rnd=None):
        """mean curvature of get_sdf_and_curvature_1d_precomputed_gradient_normal_based over the valid samples with the element-wise
        chain in three kernels (csrc/rgb_misc.cu); the SDF evaluation at the shifted points is the usual (fused) one"""
        from .fused import CurvatureLossFn, curvature_shifted_points
        shifted = curvature_shifted_points(points, sdf_gradients, rnd=rnd)
        _, grads_shifted, _ = self.get_sdf_and_gradient(shifted, iter_nr)
        return CurvatureLossFn.apply(sdf_gradients, grads_shifted, nr_valid_dev)


class RGB(torch.nn.Module, _Checkpointed):
    """models.py:309-420"""
    checkpoint_file = "rgb_model.pt"

    def __init__(self, in_channels, boundary_primitive, geom_feat_size_in, nr_iters_for_c2f, nr_levels=24, capacity=2 ** 18,
                 channels=(128, 128, 64, 3)):
        super().__init__()
        self.in_channels = in_channels
        self.boundary_primitive = boundary_primitive
        self.geom_feat_size_in = geom_feat_size_in
        self.volume_renderer_neus = VolumeRenderingNeus()
        self.encoding = make_encoding(in_channels, nr_levels, capacity, 1.0)
        self.mlp = LipshitzMLP(self.encoding.output_dims() + 25 + 3 + geom_feat_size_in, list(channels), last_layer_linear=True)
        self.c2f = permuto_enc.Coarse2Fine(nr_levels)
        self.nr_iters_for_c2f = nr_iters_for_c2f
        self.last_iter_nr = sys.maxsize
        self.fused_head = True
        self.fused = None

    def forward(self, points, samples_dirs, sdf_gradients, geom_feat, iter_nr, model_colorcal=None, img_indices=None,
                ray_start_end_idx=None):
        assert points.shape[1] == self.in_channels, "points should be N x in_channels"
        self.last_iter_nr = int(iter_nr)
        if self.fused is not None and points.is_cuda:
            # encoding + SH + normal + geom -> Lipschitz MLP in the fused tensor-core kernels (csrc/fused_rgb.cu, fused_rgb_bwd.cu)
            x = self.fused.train_forward(points, samples_dirs, sdf_gradients, geom_feat, iter_nr) if torch.is_grad_enabled() else \
                self.fused(points, samples_dirs, sdf_gradients, geom_feat, iter_nr)
            return self._head(x, model_colorcal, img_indices, ray_start_end_idx)
        window = self.c2f(map_range_val(iter_nr, 0.0, self.nr_iters_for_c2f, 0.3, 1.0))
        feat = self.encoding(points, window.view(-1))
        with torch.no_grad():
            dirs_enc = PermutoSDF.spherical_harmonics(samples_dirs, 5)
        normals = F.normalize(sdf_gradients.view(-1, 3), dim=1)
        x = torch.cat([feat, dirs_enc, normals, geom_feat], 1)
        x = self.mlp(x)
        return self._head(x, model_colorcal, img_indices, ray_start_end_idx)

    def enable_fused(self):
        """route forward / backward through the fused colour-network kernels"""
        from .fused import FusedRGB
        self.fused = FusedRGB(self)
        return self.fused

    def _head(self, x, model_colorcal, img_indices, ray_start_end_idx):
        if self.fused_head and x.is_cuda and ray_start_end_idx is not None:
            # colour calibration + sigmoid in one kernel each way (csrc/rgb_misc.cu)
            from .fused import CalibSigmoidFn
            if model_colorcal is not None:
                return CalibSigmoidFn.apply(x, ray_start_end_idx, img_indices, model_colorcal.weight_delta, model_colorcal.bias,
                                            model_colorcal.idx_with_fixed_calib)
            return CalibSigmoidFn.apply(x, ray_start_end_idx, None, None, None, -1)
        if model_colorcal is not None:
            x = model_colorcal.calib_RGB_samples_packed(x, img_indices, ray_start_end_idx)
        return torch.sigmoid(x)

    def parameters_only_encoding(self):
        return [p for n, p in self.encoding.named_parameters() if "lattice_values" in n]

    def parameters_all_without_encoding(self):
        return [p for n, p in self.named_parameters() if "lattice_values" not in n]


class NerfHash(torch.nn.Module, _Checkpointed):
    """models.py:425-563 (background model on the 4-D NeRF++ parametrisation)"""
    checkpoint_file = "nerf_hash_model.pt"

    def __init__(self, in_channels, boundary_primitive, nr_iters_for_c2f, nr_levels=24, capacity=2 ** 18):
        super().__init__()
        self.in_channels = in_channels
        self.boundary_primitive = boundary_primitive
        self.encoding = make_encoding(in_channels, nr_levels, capacity, 1.0)
        self.volume_renderer_nerf = VolumeRenderingNerf()
        self.nr_feat_for_rgb = 64
        self.mlp_feat_and_density = torch.nn.Sequential(
            torch.nn.Linear(self.encoding.output_dims(), 64), torch.nn.GELU(), torch.nn.Linear(64, 64), torch.nn.GELU(),
            torch.nn.Linear(64, 64), torch.nn.GELU(), torch.nn.Linear(64, self.nr_feat_for_rgb + 1))
        _init_stack(self.mlp_feat_and_density, last_linear_slope1=False)
        self.mlp_rgb = torch.nn.Sequential(torch.nn.Linear(self.nr_feat_for_rgb + 16, 64), torch.nn.GELU(), torch.nn.Linear(64, 64),
                                           torch.nn.GELU(), torch.nn.Linear(64, 3))
        _init_stack(self.mlp_rgb)
        self.c2f = permuto_enc.Coarse2Fine(nr_levels)
        self.nr_iters_for_c2f = nr_iters_for_c2f
        self.last_iter_nr = sys.maxsize
        self.fused = None

    def enable_fused(self):
        """route forward / backward through the fused background kernels (csrc/fused_bg.cu)"""
        from .fused import FusedNerfHash
        self.fused = FusedNerfHash(self)
        return self.fused

    def forward(self, samples_pos, samples_dirs, iter_nr, model_colorcal=None, img_indices=None, ray_start_end_idx=None):
        assert samples_pos.shape[1] == self.in_channels
        self.last_iter_nr = int(iter_nr)
        if getattr(self, "fused", None) is not None and samples_pos.is_cuda:
            rgb, density = self.fused.train_forward(samples_pos, samples_dirs, iter_nr) if torch.is_grad_enabled() else \
                self.fused(samples_pos, samples_dirs, iter_nr)
            if model_colorcal is not None:
                rgb = model_colorcal.calib_RGB_samples_packed(rgb, img_indices, ray_start_end_idx)
            return torch.sigmoid(rgb), density
        window = self.c2f(map_range_val(iter_nr, 0.0, self.nr_iters_for_c2f, 0.3, 1.0))
        feat = self.encoding(samples_pos, window.view(-1))
        with torch.no_grad():
            dirs_enc = PermutoSDF.spherical_harmonics(samples_dirs, 4)
        fd = self.mlp_feat_and_density(feat)
        density = F.softplus(fd[:, 0:1])
        rgb = self.mlp_rgb(torch.cat([F.gelu(fd[:, 1:self.nr_feat_for_rgb + 1]), dirs_enc], 1))
        if model_colorcal is not None:
            rgb = model_colorcal.calib_RGB_samples_packed(rgb, img_indices, ray_start_end_idx)
        return torch.sigmoid(rgb), density

    def get_only_density(self, ray_samples, iter_nr):
        """models.py:528-550: density [N,1] = softplus of the trunk's first output at ray_samples (reshaped to [-1, in_channels]), no
        colour head. A fused 3-D model on CUDA input runs the density-only kernel (FusedNerfHash.density, no autograd); otherwise the
        per-op encoder and trunk. Sets no last_iter_nr, as the reference does not."""
        points = ray_samples.reshape(-1, self.in_channels)
        if getattr(self, "fused", None) is not None and points.is_cuda and self.in_channels == 3:
            return self.fused.density(points, iter_nr)
        window = self.c2f(map_range_val(iter_nr, 0.0, self.nr_iters_for_c2f, 0.3, 1.0))
        fd = self.mlp_feat_and_density(self.encoding(points, window.view(-1)))
        return F.softplus(fd[:, 0:1])


class Colorcal(torch.nn.Module, _Checkpointed):
    """models.py:677-741: per-image affine colour calibration, image `idx_with_fixed_calib` stays identity"""
    checkpoint_file = "colorcal_model.pt"

    def __init__(self, nr_cams, idx_with_fixed_calib):
        super().__init__()
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        self.weight_delta = torch.nn.Parameter(torch.zeros(nr_cams, 3, device=dev))
        self.bias = torch.nn.Parameter(torch.zeros(nr_cams, 3, device=dev))
        self.idx_with_fixed_calib = idx_with_fixed_calib

    def calib_RGB_samples_packed(self, rgb_samples, per_pixel_img_indices, ray_start_end_idx):
        w = 1.0 + torch.index_select(self.weight_delta, 0, per_pixel_img_indices.long())
        b = torch.index_select(self.bias, 0, per_pixel_img_indices.long())
        fixed = per_pixel_img_indices == self.idx_with_fixed_calib
        w = torch.where(fixed[:, None], torch.ones_like(w), w)
        b = torch.where(fixed[:, None], torch.zeros_like(b), b)
        per_sample_ray_idx = RaySamplesPacked.compute_per_sample_ray_idx(ray_start_end_idx, rgb_samples.shape[0])
        return rgb_samples * torch.index_select(w, 0, per_sample_ray_idx.long()) + torch.index_select(b, 0, per_sample_ray_idx.long())
