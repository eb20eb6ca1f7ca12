"""Drop-in replacement of the external `permutohedral_encoding` package the reference imports
(permuto_sdf_py/models/models.py:20; constructor call :149, forward :186, `.output_dims()` :154,
`Coarse2Fine` :172,183). Semantics: SURVEY.md Appendix B. The device work is done by the sm_90a kernels in
csrc/encoding.cu through the C ABI (psdf_enc_forward / psdf_enc_backward / psdf_enc_double_backward).

Differentiability contract (SURVEY.md F7): out is differentiable wrt `lattice_values` and wrt `positions`;
the positions gradient itself is differentiable again wrt `lattice_values` and wrt the upstream gradient
(double backward "from positions"), which is what eikonal / curvature losses need.
"""
import math

import numpy as np
import torch

from .._lib import call


def _enc_consts(mod):
    return (mod.pos_dim, mod.nr_levels, mod.nr_feat_per_level, mod.capacity)


class _EncodeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lattice, positions, window, mod):
        D, L, F, T = _enc_consts(mod)
        N = positions.shape[0]
        out = torch.empty(N, mod.output_dims(), device=positions.device, dtype=torch.float32)
        call("psdf_enc_forward", N, D, L, F, T, positions, lattice, mod.scale_factor, mod.shift_tensor(), window,
             1 if mod.concat_points else 0, mod.concat_points_scaling, out)
        ctx.mod = mod
        ctx.save_for_backward(lattice, positions, window)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        lattice, positions, window = ctx.saved_tensors
        need_l, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        # needs_input_grad is static: torch.autograd.grad(sdf, points, create_graph=True) (models.py:245-251) also reports the
        # lattice as "needed" although its gradient is discarded. Only a backward that runs with grad mode off (loss.backward())
        # may therefore scatter straight into lattice.grad; under create_graph the table gradient goes to a scratch buffer.
        allow_in_place = not torch.is_grad_enabled()
        g_l, g_p = _EncodeBackFn.apply(lattice, positions, window, grad_out.contiguous(), ctx.mod, need_l, need_p, allow_in_place)
        if need_l and g_l.numel() == 1 and lattice.numel() != 1:
            g_l = None          # already accumulated into lattice.grad (grad_in_place)
        return (g_l if need_l else None), (g_p if need_p else None), None, None


class _EncodeBackFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lattice, positions, window, grad_out, mod, need_l, need_p, allow_in_place=True):
        D, L, F, T = _enc_consts(mod)
        N = positions.shape[0]
        # grad_in_place (flat-buffer optimizer): scatter straight into lattice.grad instead of a fresh zero-filled table
        in_place = need_l and allow_in_place and getattr(mod, "grad_in_place", False) and lattice.grad is not None and \
            lattice.grad.is_contiguous()
        g_l = (lattice.grad if in_place else torch.zeros_like(lattice)) if need_l else None
        g_p = torch.empty_like(positions) if need_p else None
        call("psdf_enc_backward", N, D, L, F, T, positions, lattice, mod.scale_factor, mod.shift_tensor(), window,
             1 if mod.concat_points else 0, mod.concat_points_scaling, grad_out, g_l, g_p)
        ctx.mod = mod
        ctx.save_for_backward(lattice, positions, window, grad_out)
        if g_l is None or in_place:
            g_l = torch.zeros(1, device=positions.device)
            ctx.mark_non_differentiable(g_l)
        if g_p is None:
            g_p = torch.zeros(1, device=positions.device)
            ctx.mark_non_differentiable(g_p)
        return g_l, g_p

    @staticmethod
    def backward(ctx, gg_lattice, gg_pos):
        # double backward is supported from the positions gradient only (like upstream)
        lattice, positions, window, grad_out = ctx.saved_tensors
        mod = ctx.mod
        D, L, F, T = _enc_consts(mod)
        N = positions.shape[0]
        need_l, need_go = ctx.needs_input_grad[0], ctx.needs_input_grad[3]
        g_l = g_go = None
        if gg_pos is not None and (need_l or need_go):
            g_l = torch.zeros_like(lattice) if need_l else None
            g_go = torch.empty_like(grad_out) if need_go else None
            call("psdf_enc_double_backward", N, D, L, F, T, positions, lattice, mod.scale_factor, mod.shift_tensor(), window,
                 1 if mod.concat_points else 0, mod.concat_points_scaling, gg_pos.contiguous(), grad_out, g_l, g_go)
        return g_l, None, None, g_go, None, None, None, None


class PermutoEncoding(torch.nn.Module):
    """PermutoEncoding(pos_dim, capacity, nr_levels, nr_feat_per_level, scale_per_level,
                       appply_random_shift_per_level=True, concat_points=False, concat_points_scaling=1.0)
    (the triple-p spelling is the upstream one, models.py:149)."""

    def __init__(self, pos_dim, capacity, nr_levels, nr_feat_per_level, scale_per_level, appply_random_shift_per_level=True,
                 concat_points=False, concat_points_scaling=1.0, dtype=torch.float32, init_scale=1e-5):
        super().__init__()
        if dtype != torch.float32:
            raise RuntimeError("only float32 lattice values are supported")
        self.pos_dim = int(pos_dim)
        self.capacity = int(capacity)
        self.nr_levels = int(nr_levels)
        self.nr_feat_per_level = int(nr_feat_per_level)
        self.scale_per_level = [float(s) for s in scale_per_level]
        if len(self.scale_per_level) != self.nr_levels:
            raise RuntimeError("scale_per_level must have nr_levels entries")
        self.apply_random_shift_per_level = bool(appply_random_shift_per_level)
        self.concat_points = bool(concat_points)
        self.concat_points_scaling = float(concat_points_scaling)
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        # upstream: randn(capacity, L, F) * 1e-5, stored as [L, capacity, F]
        lv = torch.randn(self.capacity, self.nr_levels, self.nr_feat_per_level) * init_scale
        self.lattice_values = torch.nn.Parameter(lv.permute(1, 0, 2).contiguous().to(dev))
        shift = torch.randn(self.nr_levels, self.pos_dim) * 10.0 if self.apply_random_shift_per_level else torch.zeros(
            self.nr_levels, self.pos_dim)
        self.random_shift_per_level = torch.nn.Parameter(shift.to(dev), requires_grad=False)
        # derived from scale_per_level, not state: kept out of state_dict (upstream checkpoints hold lattice_values + random shift only)
        self.register_buffer("scale_factor", self.compute_scale_factor(self.scale_per_level, self.pos_dim).to(dev), persistent=False)
        self._ones = None
        self.grad_in_place = False      # True: backward scatters into lattice_values.grad directly (set by the flat-buffer optimizer path)

    @staticmethod
    def compute_scale_factor(sigmas, pos_dim):
        # scale_factor[l][i] = 1/sqrt((i+1)(i+2)) / sigma_l   (float32 arithmetic like the upstream host code)
        sf = np.zeros((len(sigmas), pos_dim), dtype=np.float32)
        for l, s in enumerate(sigmas):
            for i in range(pos_dim):
                v = np.float32(1.0) / np.float32(math.sqrt(float((i + 1) * (i + 2))))
                sf[l, i] = np.float32(v / np.float32(s))
        return torch.from_numpy(sf)

    def shift_tensor(self):
        return self.random_shift_per_level.detach()

    def output_dims(self):
        extra = int(math.ceil(float(self.pos_dim) / self.nr_feat_per_level)) if self.concat_points else 0
        return (self.nr_levels + extra) * self.nr_feat_per_level

    def forward(self, positions, anneal_window=None):
        if positions.dim() != 2 or positions.shape[1] != self.pos_dim:
            raise RuntimeError("positions should be N x %d but is %s" % (self.pos_dim, tuple(positions.shape)))
        if not positions.is_cuda:
            raise RuntimeError("PermutoEncoding runs on CUDA tensors only (no CPU path)")
        if anneal_window is None:
            if self._ones is None or self._ones.device != positions.device:
                self._ones = torch.ones(self.nr_levels, device=positions.device)
            window = self._ones
        else:
            window = anneal_window.detach().reshape(-1).to(device=positions.device, dtype=torch.float32).contiguous()
            if window.shape[0] != self.nr_levels:
                raise RuntimeError("anneal_window should have nr_levels entries")
        pos = positions.contiguous()
        if pos.dtype != torch.float32:
            pos = pos.float()
        return _EncodeFn.apply(self.lattice_values, pos, window, self)


def cosine_easing_window(num_freqs, alpha, device=None):
    x = torch.clip(alpha - torch.arange(num_freqs, dtype=torch.float32, device=device), 0.0, 1.0)
    return 0.5 * (1 + torch.cos(math.pi * x + math.pi))


class Coarse2Fine(torch.nn.Module):
    """window_l = 0.5 (1 + cos(pi clip(t L - l, 0, 1) + pi)); remembers the last t (models.py:172,183)."""

    def __init__(self, nr_levels):
        super().__init__()
        self.nr_levels = int(nr_levels)
        self.last_t = 0
        self._cache = None

    def forward(self, t):
        self.last_t = t
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        if isinstance(t, torch.Tensor):          # device-resident schedule (CUDA-graph replay): no host read
            return cosine_easing_window(self.nr_levels, t * float(self.nr_levels), device=t.device)
        key = (float(t), str(dev))
        if self._cache is None or self._cache[0] != key:     # plateaus of the schedule: nothing to recompute
            self._cache = (key, cosine_easing_window(self.nr_levels, float(t) * self.nr_levels, device=dev))
        return self._cache[1]

    def get_last_t(self):
        return self.last_t


__all__ = ["PermutoEncoding", "Coarse2Fine", "cosine_easing_window"]
