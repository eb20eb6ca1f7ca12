"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Runs the reference's own, UNMODIFIED Python (permuto_sdf_py/models/models.py, volume_rendering/*.py, utils/sdf_utils.py, ...) on the
CPU, where a checkout of the original project is present (PERMUTO_SDF_REFERENCE, else /root/reference): `install()` puts CPU stand-ins for the two compiled modules the reference
imports into sys.modules --

  permuto_sdf            (src/PyBridge.cxx)   -> classes over the C restatement oracle/rayops_oracle.c (pinned on reference-kernel goldens)
  permutohedral_encoding (external, absent)   -> oracle/encoding_oracle.py (autograd-differentiable, parity unpinned: see its header)

-- plus empty stand-ins for the viewer / data-loader packages (easypbr, dataloaders, skimage, matplotlib, torchvision) and makes
`.cuda()` the identity. The reference classes (SDF, RGB, LipshitzMLP, NerfHash, Colorcal, VolumeRenderingNeus, ...) then import and run
as written. tests/golden/make_refpy_golden.py uses this to generate the fixtures tests/golden/refpy_*.npz that the GPU tests compare
the CUDA path with; nothing here travels to the GPU box or is imported by permuto_sdf_b200/.
"""
import math
import os
import sys
import types

import numpy as np
import torch

from . import encoding_oracle as eo
from . import rayops as ro

REF_ROOT = os.environ.get("PERMUTO_SDF_REFERENCE") or "/root/reference"


# ================================================================================================ permutohedral_encoding (CPU)
class _PermutoEncoding(torch.nn.Module):
    def __init__(self, pos_dim, capacity, nr_levels, nr_feat_per_level, scale_per_level, appply_random_shift_per_level=True,
                 concat_points=False, concat_points_scaling=1.0):
        super().__init__()
        self.pos_dim, self.capacity, self.nr_levels, self.nr_feat_per_level = int(pos_dim), int(capacity), int(nr_levels), int(nr_feat_per_level)
        self.concat_points, self.concat_points_scaling = bool(concat_points), float(concat_points_scaling)
        lv = torch.randn(self.capacity, self.nr_levels, self.nr_feat_per_level) * 1e-5
        self.lattice_values = torch.nn.Parameter(lv.permute(1, 0, 2).contiguous())
        shift = torch.randn(self.nr_levels, self.pos_dim) * 10.0 if appply_random_shift_per_level else torch.zeros(self.nr_levels, self.pos_dim)
        self.random_shift_per_level = torch.nn.Parameter(shift, requires_grad=False)
        self.scale_factor = eo.scale_factor([float(s) for s in scale_per_level], self.pos_dim)

    def output_dims(self):
        extra = int(math.ceil(float(self.pos_dim) / self.nr_feat_per_level)) if self.concat_points else 0
        return (self.nr_levels + extra) * self.nr_feat_per_level

    def forward(self, positions, anneal_window=None):
        w = None if anneal_window is None else anneal_window.detach().reshape(-1).float()
        return eo.encode(positions, self.lattice_values, self.scale_factor, self.random_shift_per_level.detach(), w, self.concat_points,
                         self.concat_points_scaling)


class _Coarse2Fine(torch.nn.Module):
    def __init__(self, nr_levels):
        super().__init__()
        self.nr_levels, self.last_t = int(nr_levels), 0

    def forward(self, t):
        self.last_t = t
        return eo.coarse2fine(self.nr_levels, t)

    def get_last_t(self):
        return self.last_t


# ================================================================================================ permuto_sdf (CPU, over the C oracle)
def _np(t):
    return None if t is None else np.ascontiguousarray(t.detach().cpu().numpy())


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


class _RaySamplesPacked:
    def __init__(self, nr_rays, nr_samples_maximum):
        M, R = int(nr_samples_maximum), int(nr_rays)
        self.samples_pos = torch.zeros(M, 3)
        self.samples_pos_4d = torch.zeros(M, 4)
        self.samples_dirs = torch.zeros(M, 3)
        self.samples_z = torch.zeros(M, 1)
        self.samples_dt = torch.zeros(M, 1)
        self.samples_sdf = torch.zeros(M, 1)
        self.ray_fixed_dt = torch.zeros(R, 1)
        self.ray_start_end_idx = torch.zeros(R, 2, dtype=torch.int32)
        self.max_nr_samples = M
        self.cur_nr_samples = torch.zeros(1, dtype=torch.int32)
        self.rays_have_equal_nr_of_samples = False
        self.fixed_nr_of_samples_per_ray = 0
        self.has_sdf = False

    # ---- oracle.rayops.Packed <-> this
    def _p(self):
        p = ro.Packed(self.ray_start_end_idx.shape[0], self.samples_z.shape[0])
        p.pos, p.dirs, p.z, p.dt, p.sdf = _np(self.samples_pos), _np(self.samples_dirs), _np(self.samples_z), _np(self.samples_dt), _np(self.samples_sdf)
        p.pos4 = _np(self.samples_pos_4d) if self.samples_pos_4d.shape[0] == self.samples_z.shape[0] else None
        p.fixed_dt, p.start_end = _np(self.ray_fixed_dt), _np(self.ray_start_end_idx).astype(np.int32)
        p.max_nr_samples, p.equal, p.fixed_n, p.has_sdf = self.samples_z.shape[0], self.rays_have_equal_nr_of_samples, self.fixed_nr_of_samples_per_ray, self.has_sdf
        return p

    @staticmethod
    def _from(p):
        r = _RaySamplesPacked(p.start_end.shape[0], p.z.shape[0])
        r.samples_pos, r.samples_dirs, r.samples_z, r.samples_dt, r.samples_sdf = _t(p.pos), _t(p.dirs), _t(p.z), _t(p.dt), _t(p.sdf)
        if p.pos4 is not None:
            r.samples_pos_4d = _t(p.pos4)
        r.ray_fixed_dt, r.ray_start_end_idx = _t(p.fixed_dt), _t(p.start_end.astype(np.int32))
        r.max_nr_samples = p.z.shape[0]
        r.cur_nr_samples = torch.tensor([int(p.cur)], dtype=torch.int32)
        r.rays_have_equal_nr_of_samples, r.fixed_nr_of_samples_per_ray, r.has_sdf = bool(p.equal), int(p.fixed_n), bool(p.has_sdf)
        return r

    def compact_to_valid_samples(self):
        return _RaySamplesPacked._from(ro.packed_compact(self._p()))

    def compute_exact_nr_samples(self):
        se = self.ray_start_end_idx
        return int((se[:, 1] - se[:, 0]).sum())

    def set_sdf(self, sdf):
        self.samples_sdf = sdf.detach().reshape(-1, 1).clone()
        self.has_sdf = True

    def remove_sdf(self):
        self.has_sdf = False

    @staticmethod
    def compute_per_sample_ray_idx(ray_start_end_idx, nr_samples):
        return _t(ro.packed_per_sample_ray_idx(_np(ray_start_end_idx).astype(np.int32), int(nr_samples)))


class _VolumeRendering:
    reference_bugs = False

    @staticmethod
    def cumprod_alpha2transmittance(rsp, alpha):
        T, bg = ro.vr_cumprod(rsp._p(), _np(alpha))
        return _t(T), _t(bg)

    @staticmethod
    def integrate_with_weights(rsp, vals, w):
        return _t(ro.vr_integrate(rsp._p(), _np(vals), _np(w)))

    @staticmethod
    def sdf2alpha(rsp, sdf, inv_s, dynamic_inv_s, inv_s_multiplier):
        return _t(ro.vr_sdf2alpha(rsp._p(), _np(sdf), float(inv_s), bool(dynamic_inv_s), float(inv_s_multiplier)))

    @staticmethod
    def sum_over_each_ray(rsp, vals):
        a, b = ro.vr_sum(rsp._p(), _np(vals))
        return _t(a), _t(b)

    @staticmethod
    def cumsum_over_each_ray(rsp, vals, inverse):
        return _t(ro.vr_cumsum(rsp._p(), _np(vals), bool(inverse)))

    @staticmethod
    def compute_cdf(rsp, w):
        return _t(ro.vr_cdf(rsp._p(), _np(w)))

    @staticmethod
    def importance_sample(origins, dirs, rsp, cdf, nr_imp, jitter):
        assert not jitter, "the CPU stand-in keeps no pcg32 stream: eval mode only"
        return _RaySamplesPacked._from(ro.vr_importance_sample(_np(origins), _np(dirs), rsp._p(), _np(cdf), int(nr_imp), False))

    @staticmethod
    def combine_uniform_samples_with_imp(origins, dirs, t_exit, rsp_uniform, rsp_imp):
        return _RaySamplesPacked._from(ro.vr_combine(_np(origins), _np(dirs), _np(t_exit), rsp_uniform._p(), rsp_imp._p()))

    @staticmethod
    def cumprod_alpha2transmittance_backward(grad_T, grad_bg, rsp, alpha, T, bg_T, cumsumLV):
        return _t(ro.vr_cumprod_backward(rsp._p(), _np(grad_bg), _np(alpha), _np(bg_T), _np(cumsumLV)))

    @staticmethod
    def integrate_with_weights_backward(g_pred, rsp, vals, w, pred):
        a, b = ro.vr_integrate_backward(rsp._p(), _np(g_pred), _np(vals), _np(w), reference_bug=True)   # the reference kernel as it is
        return _t(a), _t(b)

    @staticmethod
    def sum_over_each_ray_backward(g_ray, g_sample, rsp, vals):
        return _t(ro.vr_sum_backward(rsp._p(), _np(g_ray), _np(g_sample)))


class _PermutoSDF:
    @staticmethod
    def spherical_harmonics(dirs, degree):
        return _t(ro.spherical_harmonics(_np(dirs), int(degree)))


class _Sphere:
    def __init__(self, radius, center):
        self.m_radius = float(radius)
        self.m_center = [float(c) for c in center]
        self.m_center_tensor = torch.tensor(self.m_center)

    def ray_intersection(self, origins, dirs):
        pe, te, px, tx, hit = ro.sphere_ray_intersection(self.m_radius, np.asarray(self.m_center, np.float32), _np(origins), _np(dirs))
        return _t(pe), _t(te), _t(px), _t(tx), _t(hit)

    def check_point_inside_primitive(self, points):
        c = torch.tensor(self.m_center).view(1, 3)
        return ((points - c).norm(dim=1, keepdim=True) < self.m_radius)


class _OccupancyGrid:
    def __init__(self, V, extent, translation):
        self.V, self.extent, self.trans = int(V), float(extent), np.asarray(translation, np.float32)
        self.m_grid_values = torch.ones(self.V ** 3)
        self.m_grid_occupancy = torch.ones(self.V ** 3, dtype=torch.bool)

    def get_nr_voxels_per_dim(self):
        return self.V

    def set_grid_occupancy(self, occ):
        self.m_grid_occupancy = occ

    def get_grid_occupancy(self):
        return self.m_grid_occupancy

    def _occ(self):
        return _np(self.m_grid_occupancy).astype(np.uint8)

    def check_occupancy(self, points):
        return _t(ro.occ_check_occupancy(self.V, self.extent, self.trans, self._occ(), _np(points)))

    def compute_samples_in_occupied_regions(self, o, d, t_entry, t_exit, min_dist, max_per_ray, jitter):
        assert not jitter
        return _RaySamplesPacked._from(ro.occ_samples_in_occupied_regions(self.V, self.extent, self.trans, _np(o), _np(d), _np(t_entry),
                                                                          _np(t_exit), self._occ(), float(min_dist), int(max_per_ray), False))

    def compute_first_sample_start_of_occupied_regions(self, o, d, t_entry, t_exit):
        return _RaySamplesPacked._from(ro.occ_first_sample_start(self.V, self.extent, self.trans, _np(o), _np(d), _np(t_entry), _np(t_exit), self._occ()))

    def advance_sample_to_next_occupied_voxel(self, dirs, pos):
        p, within = ro.occ_advance_to_next_occupied(self.V, self.extent, self.trans, _np(dirs), _np(pos), self._occ())
        pos.copy_(_t(p))                    # the reference writes in place into its input (OccupancyGrid.cu:311)
        return pos, _t(within)


class _Stub:
    def __init__(self, *a, **k):
        pass


def install(ref_root=REF_ROOT):
    """-> the imported reference module permuto_sdf_py.models.models"""
    if not os.path.isdir(ref_root):
        raise RuntimeError("%r is not a checkout of the original project: set PERMUTO_SDF_REFERENCE" % ref_root)
    if "permuto_sdf_py.models.models" in sys.modules:
        return sys.modules["permuto_sdf_py.models.models"]
    for name in ("easypbr", "dataloaders", "skimage", "skimage.measure", "matplotlib", "matplotlib.cm"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["skimage"].measure = sys.modules["skimage.measure"]
    sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
    try:
        import torchvision  # noqa: F401
    except Exception:
        sys.modules["torchvision"] = types.ModuleType("torchvision")
    enc = types.ModuleType("permutohedral_encoding")
    enc.PermutoEncoding, enc.Coarse2Fine = _PermutoEncoding, _Coarse2Fine
    sys.modules["permutohedral_encoding"] = enc
    ps = types.ModuleType("permuto_sdf")
    ps.PermutoSDF, ps.RaySamplesPacked, ps.VolumeRendering, ps.Sphere, ps.OccupancyGrid = _PermutoSDF, _RaySamplesPacked, _VolumeRendering, _Sphere, _OccupancyGrid
    ps.RaySampler = ps.TrainParams = ps.NGPGui = _Stub
    sys.modules["permuto_sdf"] = ps
    torch.nn.Module.cuda = lambda self, *a, **k: self          # volume_rendering_modules.py:121 calls .cuda() in a constructor
    torch.Tensor.cuda = lambda self, *a, **k: self
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    import permuto_sdf_py.models.models as M
    return M
