"""Autograd wrappers and NeuS / NeRF weight modules of the hot path.

Mirror of permuto_sdf_py/volume_rendering/volume_rendering_funcs.py:55-223 (CumprodAlpha2TransmittanceFunc,
IntegrateWithWeightsFunc, SumOverRayFunc) and volume_rendering_modules.py:61-182 (VolumeRenderingNerf,
SingleVarianceNetwork, VolumeRenderingNeus), running on the sm_90a kernels through `permuto_sdf`.
"""
import torch
import torch.nn.functional as F
from torch.autograd import Function

from .permuto_sdf import VolumeRendering


class VolumeRenderNerfFunc(Function):
    """volume_rendering_funcs.py:14-52 (fused NeRF compositing; no gradient wrt the per-sample weights)"""

    @staticmethod
    def forward(ctx, rsp, rgb_samples, radiance_samples, ray_t_exit, use_ray_t_exit):
        pred_rgb, pred_depth, bg_T, w = VolumeRendering.volume_render_nerf(rsp, rgb_samples, radiance_samples, ray_t_exit, use_ray_t_exit)
        ctx.save_for_backward(pred_rgb, rgb_samples, radiance_samples, ray_t_exit, bg_T)
        ctx.rsp, ctx.use_ray_t_exit = rsp, use_ray_t_exit
        return pred_rgb, pred_depth, bg_T, w

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_bg, g_w):
        pred_rgb, rgb_samples, radiance_samples, ray_t_exit, bg_T = ctx.saved_tensors
        if g_w is None:
            g_w = torch.zeros_like(radiance_samples)
        if g_bg is None:
            g_bg = torch.zeros_like(bg_T)
        g_rgb_s, g_rad = VolumeRendering.volume_render_nerf_backward(g_rgb.contiguous(), g_bg.contiguous(), g_w.contiguous(), pred_rgb,
                                                                      ctx.rsp, rgb_samples, radiance_samples, ray_t_exit,
                                                                      ctx.use_ray_t_exit, bg_T)
        ctx.rsp = None
        return None, g_rgb_s, g_rad, None, None


class CumprodAlpha2TransmittanceFunc(Function):
    @staticmethod
    def forward(ctx, rsp, alpha):
        T, bg_T = VolumeRendering.cumprod_alpha2transmittance(rsp, alpha)
        ctx.save_for_backward(alpha, T, bg_T)
        ctx.rsp = rsp
        return T, bg_T

    @staticmethod
    def backward(ctx, grad_T, grad_bg):
        alpha, T, bg_T = ctx.saved_tensors
        rsp = ctx.rsp
        if grad_T is None:
            grad_T = torch.zeros_like(T)
        if grad_bg is None:
            grad_bg = torch.zeros_like(bg_T)
        cumsumLV = VolumeRendering.cumsum_over_each_ray(rsp, (grad_T * T).contiguous(), True)
        g_alpha = VolumeRendering.cumprod_alpha2transmittance_backward(grad_T.contiguous(), grad_bg.contiguous(), rsp, alpha, T, bg_T,
                                                                       cumsumLV)
        ctx.rsp = None
        return None, g_alpha


class IntegrateWithWeightsFunc(Function):
    @staticmethod
    def forward(ctx, rsp, vals, weights):
        pred = VolumeRendering.integrate_with_weights(rsp, vals, weights)
        ctx.save_for_backward(vals, weights, pred)
        ctx.rsp = rsp
        return pred

    @staticmethod
    def backward(ctx, grad_pred):
        vals, weights, pred = ctx.saved_tensors
        g_vals, g_w = VolumeRendering.integrate_with_weights_backward(grad_pred.contiguous(), ctx.rsp, vals, weights, pred)
        ctx.rsp = None
        return None, g_vals, g_w


class SumOverRayFunc(Function):
    @staticmethod
    def forward(ctx, rsp, vals):
        s_ray, s_sample = VolumeRendering.sum_over_each_ray(rsp, vals)
        ctx.save_for_backward(vals)
        ctx.rsp = rsp
        return s_ray, s_sample

    @staticmethod
    def backward(ctx, g_ray, g_sample):
        (vals,) = ctx.saved_tensors
        if g_ray is None:
            g_ray = torch.zeros(ctx.rsp.ray_start_end_idx.shape[0], vals.shape[1], device=vals.device)
        if g_sample is None:
            g_sample = torch.zeros_like(vals)
        g = VolumeRendering.sum_over_each_ray_backward(g_ray.contiguous(), g_sample.contiguous(), ctx.rsp, vals)
        ctx.rsp = None
        return None, g


class VolumeRenderingNerf(torch.nn.Module):
    """volume_rendering_modules.py:61-89"""

    def compute_weights(self, rsp, density_samples):
        dt = rsp.samples_dt
        alpha = 1.0 - torch.exp(-density_samples * dt)
        T, bg_T = CumprodAlpha2TransmittanceFunc.apply(rsp, 1 - alpha + 1e-7)
        weights = (alpha * T).view(-1, 1)
        weights_sum, _ = SumOverRayFunc.apply(rsp, weights)
        return weights, weights_sum, bg_T

    def integrate(self, rsp, vals, weights):
        return IntegrateWithWeightsFunc.apply(rsp, vals, weights)


class SingleVarianceNetwork(torch.nn.Module):
    """volume_rendering_modules.py:94-114"""

    def __init__(self, init_val):
        super().__init__()
        self.variance = torch.nn.Parameter(torch.tensor(float(init_val)))
        self.last_variance = None

    def forward(self, forced_variance=None):
        if forced_variance is not None:
            self.last_variance = forced_variance
            return torch.exp(torch.ones((), device=self.variance.device) * forced_variance * 10.0)
        self.last_variance = self.variance
        return torch.exp(self.variance * 10.0)


class VolumeRenderingNeus(torch.nn.Module):
    """volume_rendering_modules.py:116-182"""

    def __init__(self):
        super().__init__()
        self.deviation_network = SingleVarianceNetwork(init_val=0.3)
        self.last_inv_s = None

    def compute_weights(self, rsp, sdf, gradients, cos_anneal_ratio, forced_variance=None):
        dists = rsp.samples_dt
        inv_s = self.deviation_network(forced_variance).clip(1e-6, 1e6)
        self.last_inv_s = inv_s
        true_cos = (rsp.samples_dirs * gradients).sum(-1, keepdim=True)
        iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - cos_anneal_ratio) + F.relu(-true_cos) * cos_anneal_ratio)
        est_next = sdf + iter_cos * dists.reshape(-1, 1) * 0.5
        est_prev = sdf - iter_cos * dists.reshape(-1, 1) * 0.5
        prev_cdf = torch.sigmoid(est_prev * inv_s)
        next_cdf = torch.sigmoid(est_next * inv_s)
        alpha = ((prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)).clip(0.0, 1.0)
        T, bg_T = CumprodAlpha2TransmittanceFunc.apply(rsp, 1 - alpha + 1e-7)
        weights = (alpha * T).view(-1, 1)
        weights_sum, _ = SumOverRayFunc.apply(rsp, weights)
        return weights, weights_sum, bg_T, inv_s

    def integrate(self, rsp, vals, weights):
        return IntegrateWithWeightsFunc.apply(rsp, vals, weights)

    def get_last_inv_s(self):
        return self.last_inv_s.view(-1)
