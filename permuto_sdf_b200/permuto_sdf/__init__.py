"""Drop-in replacement of the reference's pybind11 module `permuto_sdf` (src/PyBridge.cxx:30-169).

Same classes, method names, argument order, tensor shapes/dtypes and aliasing semantics as the reference
(include/permuto_sdf/*.cuh), implemented on top of the C ABI of libpsdf_b200.so (include/psdf_b200.h).
Differences that are deliberate and documented in DESIGN.md:
  * tensors are created on the *current* CUDA device and kernels run on torch's current stream
    (the reference hard-codes cuda:0 and the legacy stream, src/RaySamplesPacked.cu:23);
  * shape / dtype errors raise RuntimeError instead of aborting the process (loguru CHECK);
  * sample slots are deterministic (ray-ordered) instead of atomic-ordered (SURVEY.md F8);
  * Eigen arguments are any 3-sequence.
There is no CPU path: every method needs CUDA tensors and the in-tree CUDA library.
"""
import math

import torch

from .._lib import call

_MASK64 = (1 << 64) - 1
_PCG_MULT = 0x5851F42D4C957F2D


class _Pcg32Host:
    """Host mirror of the class-static pcg32 of the reference (kernels/permuto_sdf/pcg32.h:33-34,150-171):
    copied by value into a kernel, advanced by 2^32 after every jittered call."""

    def __init__(self):
        self.state = 0x853C49E6748FEA9B
        self.inc = 0xDA3E39CB94B95BDB
        self.dev = None          # device-resident {state, inc} (int64 bit patterns) while CUDA-graph replay owns the stream

    def args(self):
        """(rng_state, rng_inc) of a C-ABI call: by value, or (device pointer, 0) for a device-resident generator"""
        if self.dev is not None:
            return self.dev.data_ptr(), 0
        return self.state, self.inc

    def to_device(self):
        """move the generator into device memory (kernels read it there; replayable from a CUDA graph)"""
        if self.dev is None:
            sg = lambda v: v - (1 << 64) if v >= (1 << 63) else v
            self.dev = torch.tensor([sg(self.state), sg(self.inc)], dtype=torch.int64, device=_dev())
        return self.dev

    def to_host(self):
        """bring a device-resident generator back (host sync)"""
        if self.dev is not None:
            st = self.dev.cpu().tolist()
            self.state, self.inc = st[0] & _MASK64, st[1] & _MASK64
            self.dev = None

    def advance(self, delta=1 << 32):
        if self.dev is not None:
            call("psdf_rng_advance_dev", self.dev, int(delta))
            return
        cur_mult, cur_plus, acc_mult, acc_plus = _PCG_MULT, self.inc, 1, 0
        delta &= _MASK64
        while delta > 0:
            if delta & 1:
                acc_mult = (acc_mult * cur_mult) & _MASK64
                acc_plus = (acc_plus * cur_mult + cur_plus) & _MASK64
            cur_plus = ((cur_mult + 1) * cur_plus) & _MASK64
            cur_mult = (cur_mult * cur_mult) & _MASK64
            delta >>= 1
        self.state = (acc_mult * self.state + acc_plus) & _MASK64


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _f32(t, name, cols=None):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda:
        raise RuntimeError("%s must be a float32 CUDA tensor" % name)
    if cols is not None and (t.dim() != 2 or t.shape[1] != cols):
        raise RuntimeError("%s should have shape [n,%d] but has %s" % (name, cols, tuple(t.shape)))
    return t.contiguous()


# ======================================================================================================
class RaySamplesPacked:
    """include/permuto_sdf/RaySamplesPacked.cuh:7-46, src/RaySamplesPacked.cu:19-155

    `RaySamplesPacked.static_capacity = True` switches compaction to a sync-free mode: compact_to_valid_samples keeps the
    capacity of its input (valid samples packed at the front, zero-filled tail, exact count only in the device tensor
    cur_nr_samples), so that every tensor shape of an iteration is known on the host and the iteration can be captured in a
    CUDA graph. The default (False) sizes the compacted container exactly, with the reference's host sync."""
    static_capacity = False

    def __init__(self, nr_rays, nr_samples_maximum, zero=False, zero_count=True):
        d = _dev()
        self.m_nr_rays = int(nr_rays)
        self.max_nr_samples = int(nr_samples_maximum)
        M = self.max_nr_samples
        self.is_compact = False
        # the samplers add into the counter (it must start at zero); compaction / merge / resampling overwrite or ignore it
        self.cur_nr_samples = torch.zeros(1, dtype=torch.int32, device=d) if zero_count else torch.empty(1, dtype=torch.int32, device=d)
        if zero:
            # one zero-filled arena (a single memset) carved into the per-sample arrays; offsets keep 16-byte alignment
            Mp = (M + 3) // 4 * 4
            arena = torch.zeros(9 * Mp, device=d)
            self.samples_pos = arena[0:3 * M].view(M, 3)
            self.samples_dirs = arena[3 * Mp:3 * Mp + 3 * M].view(M, 3)
            self.samples_z = arena[6 * Mp:6 * Mp + M].view(M, 1)
            self.samples_dt = arena[7 * Mp:7 * Mp + M].view(M, 1)
            self._zero_sdf = arena[8 * Mp:8 * Mp + M].view(M, 1)
        else:
            self.samples_pos = torch.empty(M, 3, device=d)
            self.samples_dirs = torch.empty(M, 3, device=d)
            self.samples_z = torch.empty(M, 1, device=d)
            self.samples_dt = torch.empty(M, 1, device=d)
            self._zero_sdf = None
        self._samples_pos_4d = None   # allocated on first use (only background containers need it)
        self._samples_sdf = None
        self.ray_fixed_dt = torch.empty(self.m_nr_rays, 1, device=d)
        self.ray_start_end_idx = torch.empty(self.m_nr_rays, 2, dtype=torch.int32, device=d)
        self.rays_have_equal_nr_of_samples = False
        self.fixed_nr_of_samples_per_ray = 0
        self.has_sdf = False

    # lazily materialised members keep the reference attribute names
    @property
    def samples_pos_4d(self):
        if self._samples_pos_4d is None:
            self._samples_pos_4d = torch.empty(self.samples_z.shape[0], 4, device=self.samples_z.device)
        return self._samples_pos_4d

    @samples_pos_4d.setter
    def samples_pos_4d(self, v):
        self._samples_pos_4d = v

    @property
    def samples_sdf(self):
        if self._samples_sdf is None:
            self._samples_sdf = torch.empty(self.samples_z.shape[0], 1, device=self.samples_z.device)
        return self._samples_sdf

    @samples_sdf.setter
    def samples_sdf(self, v):
        self._samples_sdf = v

    def compute_exact_nr_samples(self):
        total = torch.empty(1, dtype=torch.int32, device=self.ray_start_end_idx.device)
        call("psdf_packed_count_samples", self.m_nr_rays, self.ray_start_end_idx, total)
        return int(total.item())

    def compact_to_valid_samples(self):
        R = self.m_nr_rays
        d = self.ray_start_end_idx.device
        static = RaySamplesPacked.static_capacity
        if static and self.is_compact:
            return self
        nblocks = (max(R, 1) + 1023) // 1024
        ws = torch.empty(R + nblocks + 1, dtype=torch.int32, device=d)
        se = self.ray_start_end_idx.contiguous()
        if R > 0:
            call("psdf_packed_compact_scan", R, se, ws)
            # exact size: the reference's host sync (RaySamplesPacked.cu:51); static mode keeps the capacity instead
            exact = self.max_nr_samples if static else int(ws[R + nblocks].item())
        else:
            exact = 0
        out = RaySamplesPacked(R, exact, zero=static, zero_count=False)
        out.is_compact = True
        out.has_sdf = self.has_sdf
        out.rays_have_equal_nr_of_samples = self.rays_have_equal_nr_of_samples
        out.fixed_nr_of_samples_per_ray = self.fixed_nr_of_samples_per_ray
        if static and R > 0:
            out.cur_nr_samples = ws[R + nblocks:R + nblocks + 1]
            if self._samples_pos_4d is not None:
                out._samples_pos_4d = torch.zeros(exact, 4, device=d)
            if self._samples_sdf is not None:
                out._samples_sdf = out._zero_sdf
        else:
            out.cur_nr_samples.fill_(exact)
        if R > 0:
            pos4 = self._samples_pos_4d
            sdf = self._samples_sdf if self._samples_sdf is not None else None
            call("psdf_packed_compact_copy", R, self.samples_pos.reshape(-1, 3), None if pos4 is None else pos4.reshape(-1, 4),
                 self.samples_dirs.reshape(-1, 3), self.samples_z.reshape(-1, 1), self.samples_dt.reshape(-1, 1),
                 None if sdf is None else sdf.reshape(-1, 1).contiguous(), self.ray_fixed_dt, se, ws,
                 out.samples_pos, None if pos4 is None else out.samples_pos_4d, out.samples_dirs, out.samples_z,
                 out.samples_dt, None if sdf is None else out.samples_sdf, out.ray_fixed_dt, out.ray_start_end_idx)
        return out

    def initialize_with_one_sample_per_ray(self, one_sample_per_ray, dirs):
        n = one_sample_per_ray.shape[0]
        d = one_sample_per_ray.device
        self.samples_pos = one_sample_per_ray
        self.samples_dirs = dirs
        self.samples_z = torch.zeros(n, 1, device=d)
        self.samples_dt = torch.zeros(n, 1, device=d)
        self.ray_fixed_dt = torch.zeros(n, 1, device=d)
        start = torch.arange(n, dtype=torch.int32, device=d).view(-1, 1)
        self.ray_start_end_idx = torch.cat([start, start + 1], 1).contiguous()
        self.max_nr_samples = n
        self.cur_nr_samples.fill_(n)
        self.rays_have_equal_nr_of_samples = True
        self.fixed_nr_of_samples_per_ray = 1
        self.has_sdf = False

    def set_sdf(self, sdf):
        self._samples_sdf = sdf.view(-1, 1)
        self.has_sdf = True

    def remove_sdf(self):
        self.has_sdf = False

    @staticmethod
    def compute_per_sample_ray_idx(ray_start_end_idx, nr_samples):
        R = ray_start_end_idx.shape[0]
        # rows outside every ray keep index 0 (a valid row for downstream gathers)
        out = torch.zeros(int(nr_samples), dtype=torch.int32, device=ray_start_end_idx.device)
        call("psdf_packed_per_sample_ray_idx", R, int(nr_samples), ray_start_end_idx.contiguous(), out)
        return out

    # helper for the volume-rendering calls
    def _rsp(self):
        return (self.ray_start_end_idx.shape[0], self.max_nr_samples, self.ray_start_end_idx,
                1 if self.rays_have_equal_nr_of_samples else 0, self.fixed_nr_of_samples_per_ray)


# ======================================================================================================
class Sphere:
    """include/permuto_sdf/Sphere.cuh:12-24, src/Sphere.cu"""

    def __init__(self, radius, center):
        self.m_radius = float(radius)
        self.m_center = [float(c) for c in center]
        self.m_center_tensor = torch.tensor(self.m_center, dtype=torch.float32, device=_dev())

    def ray_intersection(self, ray_origins, ray_dirs):
        if ray_origins.dim() != 2 or ray_dirs.dim() != 2:
            raise RuntimeError("ray_origins / ray_dirs should have dim 2 corresponding to nr_rays x 3")
        o, dr = _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3)
        n, d = o.shape[0], o.device
        pe = torch.empty(n, 3, device=d); te = torch.empty(n, 1, device=d)
        px = torch.empty(n, 3, device=d); tx = torch.empty(n, 1, device=d)
        hit = torch.empty(n, 1, dtype=torch.bool, device=d)
        call("psdf_sphere_ray_intersection", n, self.m_radius, self.m_center, o, dr, pe, te, px, tx, hit)
        return pe, te, px, tx, hit

    def rand_points_inside(self, nr_points):
        d = self.m_center_tensor.device
        n = int(nr_points)
        phi = torch.empty(n, device=d).uniform_(0, 2 * math.pi)
        costheta = torch.empty(n, device=d).uniform_(-1, 1)
        u = torch.rand(n, device=d)
        pts = torch.empty(n, 3, device=d)
        call("psdf_sphere_rand_points_inside", n, self.m_radius, phi, costheta, u, pts)
        return pts

    def rand_points_inside_u01(self, u01):
        """rand_points_inside from ONE uniform draw u01 [3,n] in [0,1) (rows: phi / 2 pi, (cos theta + 1) / 2, u): one RNG launch and one
        kernel instead of three and one (not in the reference; used by the training iteration for its off-surface points)"""
        u = _f32(u01, "u01").contiguous()
        n = u.shape[1]
        pts = torch.empty(n, 3, device=u.device)
        call("psdf_sphere_rand_points_inside_u01", n, self.m_radius, u, pts)
        return pts

    def check_point_inside_primitive(self, points):
        p = _f32(points, "points", 3)
        out = torch.empty(p.shape[0], 1, dtype=torch.bool, device=p.device)
        call("psdf_sphere_check_point_inside", p.shape[0], self.m_radius, self.m_center, p, out)
        return out


# ======================================================================================================
class AABB:
    """permuto_sdf_py/utils/aabb.py:8-114: the axis-aligned bounding box of train_sdf_from_mesh.py, the SDF model's boundary_primitive
    there (sizes and translation are 3-sequences). The sphere tracer and the samplers of this package take a bounding Sphere."""

    def __init__(self, bounding_box_sizes_xyz, bounding_box_translation):
        self.bounding_box_sizes_xyz = [float(v) for v in bounding_box_sizes_xyz]
        self.bounding_box_translation = [float(v) for v in bounding_box_translation]
        if len(self.bounding_box_sizes_xyz) != 3 or len(self.bounding_box_translation) != 3:
            raise RuntimeError("AABB: sizes and translation must have 3 components")
        half = [s / 2 for s in self.bounding_box_sizes_xyz]
        self.max_bounds = torch.tensor(half)
        self.min_bounds = torch.tensor([-h for h in half])

    def check_point_inside_primitive(self, points):
        """[N,3] -> [N,1] bool: every coordinate strictly inside the box (aabb.py:28-43)"""
        d = points.device
        p = points - torch.as_tensor(self.bounding_box_translation, device=d)
        inside = torch.logical_and(p < self.max_bounds.to(d), p > self.min_bounds.to(d))
        return (inside * 1.0).sum(dim=-1, keepdim=True) == 3

    def rand_points_inside(self, nr_points):
        """nr_points uniform points in the box (aabb.py:110-114): one torch.rand(nr_points, 3) draw, then rand_points_inside_u01"""
        return self.rand_points_inside_u01(torch.rand(int(nr_points), 3, device=_dev()))

    def rand_points_inside_u01(self, u01):
        """the box points of a given uniform draw u01 [n,3]: u01 * size - size / 2 + translation, bit-identical to the reference's
        expression (one kernel, psdf_surface_fit_points without cloud rows)"""
        u = _f32(u01, "u01", 3)
        out = torch.empty(u.shape[0], 3, device=u.device)
        call("psdf_surface_fit_points", 0, 0, u.shape[0], None, None, None, u, self.bounding_box_sizes_xyz, self.bounding_box_translation,
             out, None)
        return out


# ======================================================================================================
class OccupancyGrid:
    """include/permuto_sdf/OccupancyGrid.cuh:19-64, src/OccupancyGrid.cu"""

    m_rng = _Pcg32Host()

    def __init__(self, nr_voxels_per_dim, grid_extent, grid_translation):
        self.m_nr_voxels_per_dim = int(nr_voxels_per_dim)
        self.m_grid_extent = float(grid_extent)
        self.m_grid_translation = [float(c) for c in grid_translation]
        self.m_grid_translation_tensor = torch.tensor(self.m_grid_translation, dtype=torch.float32, device=_dev())
        self.m_grid_values = OccupancyGrid.make_grid_values(self.m_nr_voxels_per_dim)
        self.m_grid_occupancy = OccupancyGrid.make_grid_occupancy(self.m_nr_voxels_per_dim)

    @staticmethod
    def _check_v(v):
        if v % 2 != 0 or (v & (v - 1)) != 0 or v > 1024:
            raise RuntimeError("nr_voxels_per_dim must be a power of two <= 1024 (Morton codes)")

    @staticmethod
    def make_grid_values(nr_voxels_per_dim):
        OccupancyGrid._check_v(nr_voxels_per_dim)
        return torch.ones(nr_voxels_per_dim ** 3, dtype=torch.float32, device=_dev())

    @staticmethod
    def make_grid_occupancy(nr_voxels_per_dim):
        OccupancyGrid._check_v(nr_voxels_per_dim)
        return torch.ones(nr_voxels_per_dim ** 3, dtype=torch.bool, device=_dev())

    def get_nr_voxels(self):
        return self.m_nr_voxels_per_dim ** 3

    def get_nr_voxels_per_dim(self):
        return self.m_nr_voxels_per_dim

    def get_grid_values(self):
        return self.m_grid_values

    def get_grid_occupancy(self):
        return self.m_grid_occupancy

    def set_grid_values(self, grid_values):
        self.m_grid_values = grid_values

    def set_grid_occupancy(self, grid_occupancy):
        self.m_grid_occupancy = grid_occupancy

    def _geom(self):
        return self.m_nr_voxels_per_dim, self.m_grid_extent, self.m_grid_translation

    def compute_grid_points(self, randomize_position):
        n = self.get_nr_voxels()
        out = torch.empty(n, 3, device=self.m_grid_values.device)
        V, e, t = self._geom()
        call("psdf_occ_compute_grid_points", n, V, e, t, None, *OccupancyGrid.m_rng.args(),
             1 if randomize_position else 0, out)
        if randomize_position:
            OccupancyGrid.m_rng.advance()
        return out

    def compute_random_sample_of_grid_points(self, nr_voxels_to_select, randomize_position):
        n = int(nr_voxels_to_select)
        d = self.m_grid_values.device
        out = torch.empty(n, 3, device=d)
        idx = torch.randint(0, self.get_nr_voxels(), (n,), dtype=torch.int32, device=d)
        V, e, t = self._geom()
        call("psdf_occ_compute_grid_points", n, V, e, t, idx, *OccupancyGrid.m_rng.args(),
             1 if randomize_position else 0, out)
        if randomize_position:
            OccupancyGrid.m_rng.advance()
        return out, idx

    def check_occupancy(self, points):
        p = _f32(points, "points", 3)
        out = torch.empty(p.shape[0], 1, dtype=torch.bool, device=p.device)
        V, e, t = self._geom()
        call("psdf_occ_check_occupancy", p.shape[0], V, e, t, self.m_grid_occupancy, p, out)
        return out

    def update_with_density(self, density, decay, occupancy_tresh):
        if density.dim() != 2:
            raise RuntimeError("density should have dim 2 corresponding to nr_points x 1")
        if not decay < 1.0:
            raise RuntimeError("We expect the decay to be < 1.0 but it is %f" % decay)
        call("psdf_occ_update_with_density", self.get_nr_voxels(), _f32(density, "density"), None, decay, occupancy_tresh,
             self.m_grid_values, self.m_grid_occupancy)

    def update_with_density_random_sample(self, point_indices, density, decay, occupancy_tresh):
        if density.dim() != 2 or point_indices.dim() != 1:
            raise RuntimeError("density should be nr_points x 1 and point_indices nr_points")
        if not decay < 1.0:
            raise RuntimeError("We expect the decay to be < 1.0 but it is %f" % decay)
        call("psdf_occ_update_with_density", point_indices.shape[0], _f32(density, "density"), point_indices.contiguous(),
             decay, occupancy_tresh, self.m_grid_values, self.m_grid_occupancy)

    def update_with_sdf(self, sdf, inv_s, max_eikonal_abs, occupancy_thresh):
        if sdf.dim() != 2:
            raise RuntimeError("sdf should have dim 2 corresponding to nr_points x 1")
        call("psdf_occ_update_with_sdf", self.get_nr_voxels(), _f32(sdf, "sdf"), None, self.m_grid_extent,
             self.m_nr_voxels_per_dim, float(inv_s), None, occupancy_thresh, 0, self.m_grid_values, self.m_grid_occupancy)

    def update_with_sdf_random_sample(self, point_indices, sdf, inv_s, occupancy_thresh):
        if sdf.dim() != 2 or point_indices.dim() != 1:
            raise RuntimeError("sdf should be nr_points x 1 and point_indices nr_points")
        if not isinstance(inv_s, torch.Tensor) or inv_s.dim() != 1 or inv_s.shape[0] != 1:
            raise RuntimeError("inv_s should be a tensor of 1 element")
        call("psdf_occ_update_with_sdf", point_indices.shape[0], _f32(sdf, "sdf"), point_indices.contiguous(),
             self.m_grid_extent, self.m_nr_voxels_per_dim, 0.0, _f32(inv_s.detach(), "inv_s"), occupancy_thresh, 1,
             self.m_grid_values, self.m_grid_occupancy)

    def compute_samples_in_occupied_regions(self, ray_origins, ray_dirs, ray_t_entry, ray_t_exit, min_dist_between_samples,
                                            max_nr_samples_per_ray, jitter_samples):
        o, dr = _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3)
        R = o.shape[0]
        # the reference reserves a fixed 2*1024*1024 pool (OccupancyGrid.cu:216); ray-strided slots need R*max
        M = max(R * int(max_nr_samples_per_ray), 1)
        rsp = RaySamplesPacked(R, M)
        V, e, t = self._geom()
        call("psdf_occ_compute_samples_in_occupied_regions", R, V, e, t, o, dr, _f32(ray_t_entry, "t_entry"),
             _f32(ray_t_exit, "t_exit"), self.m_grid_occupancy, float(min_dist_between_samples), int(max_nr_samples_per_ray), M,
             *OccupancyGrid.m_rng.args(), 1 if jitter_samples else 0, 1, rsp.samples_pos,
             rsp.samples_dirs, rsp.samples_z, rsp.samples_dt, rsp.ray_fixed_dt, rsp.ray_start_end_idx, rsp.cur_nr_samples)
        if jitter_samples:
            OccupancyGrid.m_rng.advance()
        return rsp

    def compute_first_sample_start_of_occupied_regions(self, ray_origins, ray_dirs, ray_t_entry, ray_t_exit):
        o, dr = _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3)
        R = o.shape[0]
        rsp = RaySamplesPacked(R, max(R, 1))
        V, e, t = self._geom()
        call("psdf_occ_compute_first_sample_start", R, V, e, t, o, dr, _f32(ray_t_entry, "t_entry"), _f32(ray_t_exit, "t_exit"),
             self.m_grid_occupancy, max(R, 1), 1, rsp.samples_pos, rsp.samples_dirs, rsp.samples_z, rsp.samples_dt,
             rsp.ray_fixed_dt, rsp.ray_start_end_idx, rsp.cur_nr_samples)
        return rsp

    def advance_sample_to_next_occupied_voxel(self, samples_dirs, samples_pos):
        dr = _f32(samples_dirs, "samples_dirs", 3)
        if not samples_pos.is_contiguous():
            raise RuntimeError("samples_pos must be contiguous (it is updated in place, like the reference)")
        n = samples_pos.shape[0]
        within = torch.ones(n, 1, dtype=torch.bool, device=samples_pos.device)
        V, e, t = self._geom()
        call("psdf_occ_advance_sample_to_next_occupied_voxel", n, V, e, t, dr, samples_pos, self.m_grid_occupancy, within)
        return samples_pos, within

    def create_cubes_for_occupied_voxels(self):
        raise RuntimeError("create_cubes_for_occupied_voxels needs EasyPBR (debug viewer only); out of scope")


# ======================================================================================================
class RaySampler:
    """include/permuto_sdf/RaySampler.cuh:21-22, src/RaySampler.cu"""

    m_rng = _Pcg32Host()

    @staticmethod
    def compute_samples_bg(ray_origins, ray_dirs, ray_t_exit, nr_samples_per_ray, sphere_radius, sphere_center,
                           randomize_position, contract_3d_samples):
        o, dr = _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3)
        R, n = o.shape[0], int(nr_samples_per_ray)
        rsp = RaySamplesPacked(R, R * n)
        rsp.rays_have_equal_nr_of_samples = True
        rsp.fixed_nr_of_samples_per_ray = n
        c = sphere_center.tolist() if isinstance(sphere_center, torch.Tensor) else list(sphere_center)
        call("psdf_sampler_bg", R, n, o, dr, _f32(ray_t_exit, "ray_t_exit"), float(sphere_radius), c, *RaySampler.m_rng.args(), 1 if randomize_position else 0, 1 if contract_3d_samples else 0, rsp.samples_pos,
             rsp.samples_pos_4d, rsp.samples_dirs, rsp.samples_z, rsp.samples_dt, rsp.ray_fixed_dt, rsp.ray_start_end_idx)
        if randomize_position:
            RaySampler.m_rng.advance()
        rsp.cur_nr_samples.fill_(R * n)
        return rsp

    @staticmethod
    def compute_samples_fg(ray_origins, ray_dirs, ray_t_entry, ray_t_exit, min_dist_between_samples, max_nr_samples_per_ray,
                           sphere_radius, sphere_center, randomize_position):
        o, dr = _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3)
        R = o.shape[0]
        M = max(R * int(max_nr_samples_per_ray), 1)
        rsp = RaySamplesPacked(R, M)
        call("psdf_sampler_fg", R, o, dr, _f32(ray_t_entry, "t_entry"), _f32(ray_t_exit, "t_exit"),
             float(min_dist_between_samples), int(max_nr_samples_per_ray), M, *RaySampler.m_rng.args(),
             1 if randomize_position else 0, 1, rsp.samples_pos, rsp.samples_dirs, rsp.samples_z, rsp.samples_dt,
             rsp.ray_fixed_dt, rsp.ray_start_end_idx, rsp.cur_nr_samples)
        if randomize_position:
            RaySampler.m_rng.advance()
        return rsp


# ======================================================================================================
class VolumeRendering:
    """include/permuto_sdf/VolumeRendering.cuh:22-38, src/VolumeRendering.cu (all static)"""

    m_rng = _Pcg32Host()
    # reproduce the green-for-blue read of integrate_with_weights_backward (VolumeRenderingGPU.cuh:1247)?
    reference_bugs = False

    @staticmethod
    def _N(rsp):
        return rsp.samples_z.shape[0]

    @staticmethod
    def cumprod_alpha2transmittance(rsp, alpha_samples):
        N, R = VolumeRendering._N(rsp), rsp.ray_start_end_idx.shape[0]
        d = rsp.samples_z.device
        T = torch.zeros(N, 1, device=d)
        bg = torch.ones(R, 1, device=d)
        call("psdf_vr_cumprod_alpha2transmittance", *rsp._rsp(), _f32(alpha_samples, "alpha"), T, bg)
        return T, bg

    @staticmethod
    def integrate_with_weights(rsp, rgb_samples, weights_samples):
        R = rsp.ray_start_end_idx.shape[0]
        out = torch.zeros(R, 3, device=rsp.samples_z.device)
        call("psdf_vr_integrate_with_weights", *rsp._rsp(), _f32(rgb_samples, "vals", 3), _f32(weights_samples, "weights"), out)
        return out

    @staticmethod
    def sdf2alpha(rsp, sdf_samples, inv_s, dynamic_inv_s, inv_s_multiplier):
        N = VolumeRendering._N(rsp)
        alpha = torch.zeros(N, 1, device=rsp.samples_z.device)
        call("psdf_vr_sdf2alpha", *rsp._rsp(), rsp.ray_fixed_dt, rsp.samples_dt, _f32(sdf_samples, "sdf"), float(inv_s),
             1 if dynamic_inv_s else 0, float(inv_s_multiplier), alpha)
        return alpha

    @staticmethod
    def sum_over_each_ray(rsp, sample_values):
        N, R = VolumeRendering._N(rsp), rsp.ray_start_end_idx.shape[0]
        v = _f32(sample_values, "sample_values")
        if v.shape[0] != N:
            raise RuntimeError("sample_values should have size nr_samples_total x c but has %s" % (tuple(v.shape),))
        D = v.shape[1]
        if not (D <= 3 or D == 32):
            raise RuntimeError("sample_values should have 1, 2, 3 or 32 values per sample")
        d = v.device
        s_ray = torch.zeros(R, D, device=d)
        s_smp = torch.zeros(N, D, device=d)
        call("psdf_vr_sum_over_each_ray", *rsp._rsp(), D, v, s_ray, s_smp)
        return s_ray, s_smp

    @staticmethod
    def cumsum_over_each_ray(rsp, sample_values, inverse):
        N = VolumeRendering._N(rsp)
        v = _f32(sample_values, "sample_values", 1)
        if v.shape[0] != N:
            raise RuntimeError("sample_values should have size nr_samples_total x 1")
        out = torch.zeros(N, 1, device=v.device)
        call("psdf_vr_cumsum_over_each_ray", *rsp._rsp(), v, 1 if inverse else 0, out)
        return out

    @staticmethod
    def compute_cdf(rsp, sample_weights):
        N = VolumeRendering._N(rsp)
        w = _f32(sample_weights, "sample_weights", 1)
        if w.shape[0] != N:
            raise RuntimeError("Weights should have size nr_samples_total x 1")
        cdf = torch.zeros(N, 1, device=w.device)
        call("psdf_vr_compute_cdf", *rsp._rsp(), w, cdf)
        return cdf

    @staticmethod
    def importance_sample(ray_origins, ray_dirs, rsp, sample_cdf, nr_importance_samples, jitter_samples):
        R = rsp.ray_start_end_idx.shape[0]
        k = int(nr_importance_samples)
        imp = RaySamplesPacked(R, R * k, zero_count=False)
        imp.rays_have_equal_nr_of_samples = True
        imp.fixed_nr_of_samples_per_ray = k
        call("psdf_vr_importance_sample", *rsp._rsp(), _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3),
             rsp.ray_fixed_dt, rsp.samples_z, _f32(sample_cdf, "cdf", 1), k, *VolumeRendering.m_rng.args(), 1 if jitter_samples else 0, imp.samples_pos, imp.samples_dirs, imp.samples_z)
        if jitter_samples:
            VolumeRendering.m_rng.advance()
        return imp

    @staticmethod
    def importance_round(ray_origins, ray_dirs, rsp, sdf_samples, inv_s, dynamic_inv_s, inv_s_multiplier, nr_importance_samples,
                         jitter_samples):
        """sdf2alpha -> clip -> cumprod_alpha2transmittance -> weights -> normalise -> compute_cdf -> importance_sample in one launch
        (one round of importance_sampling_sdf_model); bit-identical to the separate calls, same generator use"""
        R = rsp.ray_start_end_idx.shape[0]
        k = int(nr_importance_samples)
        imp = RaySamplesPacked(R, R * k, zero_count=False)
        imp.rays_have_equal_nr_of_samples = True
        imp.fixed_nr_of_samples_per_ray = k
        cdf = torch.empty(VolumeRendering._N(rsp), 1, device=rsp.samples_z.device)      # scratch: every entry is written before it is read
        call("psdf_vr_importance_round", *rsp._rsp(), _f32(ray_origins, "ray_origins", 3), _f32(ray_dirs, "ray_dirs", 3), rsp.ray_fixed_dt,
             rsp.samples_dt, rsp.samples_z, _f32(sdf_samples, "sdf").reshape(-1, 1), float(inv_s), 1 if dynamic_inv_s else 0,
             float(inv_s_multiplier), k, *VolumeRendering.m_rng.args(), 1 if jitter_samples else 0, cdf, imp.samples_pos, imp.samples_dirs,
             imp.samples_z)
        if jitter_samples:
            VolumeRendering.m_rng.advance()
        return imp

    @staticmethod
    def combine_uniform_samples_with_imp(ray_origins, ray_dirs, ray_t_exit, rsp, rsp_imp):
        if not rsp_imp.rays_have_equal_nr_of_samples:
            raise RuntimeError("importance samples are expected to have an equal nr of samples per ray")
        if rsp.has_sdf != rsp_imp.has_sdf:
            raise RuntimeError("both containers are supposed to have, or not have, sdf")
        R = rsp.ray_start_end_idx.shape[0]
        k = rsp_imp.fixed_nr_of_samples_per_ray
        c_max = VolumeRendering._N(rsp) + R * k
        comb = RaySamplesPacked(R, max(c_max, 1), zero=RaySamplesPacked.static_capacity, zero_count=False)
        comb.is_compact = True          # the merge writes ray after ray at the scanned offsets
        if RaySamplesPacked.static_capacity and rsp.has_sdf:
            comb._samples_sdf = comb._zero_sdf
        comb.has_sdf = rsp.has_sdf
        nblocks = (max(R, 1) + 1023) // 1024
        ws = torch.empty(R + nblocks + 1, dtype=torch.int32, device=rsp.samples_z.device)
        call("psdf_vr_combine_uniform_samples_with_imp", *rsp._rsp(), _f32(ray_origins, "ray_origins", 3),
             _f32(ray_dirs, "ray_dirs", 3), _f32(ray_t_exit, "ray_t_exit"), rsp.ray_fixed_dt, rsp.samples_z,
             rsp.samples_sdf.contiguous() if rsp.has_sdf else None, 1 if rsp.has_sdf else 0, k, rsp_imp.samples_z,
             rsp_imp.samples_sdf.contiguous() if rsp_imp.has_sdf else None, 1 if rsp_imp.has_sdf else 0, max(c_max, 1), ws,
             comb.samples_pos, comb.samples_dirs, comb.samples_z, comb.samples_dt, comb.samples_sdf if rsp.has_sdf else None,
             comb.ray_fixed_dt, comb.ray_start_end_idx)
        comb.cur_nr_samples = ws[R + nblocks:R + nblocks + 1]
        return comb

    @staticmethod
    def cumprod_alpha2transmittance_backward(grad_transmittance, grad_bg_transmittance, rsp, alpha, transmittance,
                                             bg_transmittance, cumsumLV):
        N = VolumeRendering._N(rsp)
        if grad_transmittance.shape[0] != N:
            raise RuntimeError("grad_transmittance should have size nr_samples_total x 1")
        g = torch.zeros(N, 1, device=alpha.device)
        call("psdf_vr_cumprod_alpha2transmittance_backward", *rsp._rsp(), _f32(grad_bg_transmittance, "grad_bg"),
             _f32(alpha, "alpha"), _f32(bg_transmittance, "bg_T"), _f32(cumsumLV, "cumsumLV"), g)
        return g

    @staticmethod
    def integrate_with_weights_backward(grad_pred_rgb, rsp, rgb_samples, weights_samples, pred_rgb):
        N, R = VolumeRendering._N(rsp), rsp.ray_start_end_idx.shape[0]
        if grad_pred_rgb.shape[0] != R or grad_pred_rgb.shape[1] != 3:
            raise RuntimeError("grad_pred_rgb should have size nr_rays x 3")
        d = rgb_samples.device
        g_rgb = torch.zeros(N, 3, device=d)
        g_w = torch.zeros(N, 1, device=d)
        call("psdf_vr_integrate_with_weights_backward", *rsp._rsp(), _f32(grad_pred_rgb, "grad_pred_rgb"),
             _f32(rgb_samples, "vals", 3), _f32(weights_samples, "weights"), 1 if VolumeRendering.reference_bugs else 0, g_rgb, g_w)
        return g_rgb, g_w

    @staticmethod
    def sum_over_each_ray_backward(grad_values_sum_per_ray, grad_values_sum_per_sample, rsp, sample_values):
        N, R = VolumeRendering._N(rsp), rsp.ray_start_end_idx.shape[0]
        D = sample_values.shape[1]
        if grad_values_sum_per_ray.shape[0] != R or grad_values_sum_per_sample.shape[0] != N:
            raise RuntimeError("bad gradient shapes for sum_over_each_ray_backward")
        g = torch.zeros(N, D, device=sample_values.device)
        call("psdf_vr_sum_over_each_ray_backward", *rsp._rsp(), D, _f32(grad_values_sum_per_ray, "g_ray"),
             _f32(grad_values_sum_per_sample, "g_sample"), g)
        return g

    @staticmethod
    def compute_dt(rsp, ray_t_exit, use_ray_t_exit):
        N = VolumeRendering._N(rsp)
        dt = torch.zeros(N, 1, device=rsp.samples_z.device)
        call("psdf_vr_compute_dt", *rsp._rsp(), 1 if use_ray_t_exit else 0, _f32(ray_t_exit, "ray_t_exit"), rsp.samples_z, dt)
        return dt

    @staticmethod
    def volume_render_nerf(rsp, rgb_samples, radiance_samples, ray_t_exit, use_ray_t_exit):
        if rgb_samples.dim() != 2 or radiance_samples.dim() != 2:
            raise RuntimeError("rgb_samples / radiance_samples should be nr_samples x 3 / x 1")
        N, R = VolumeRendering._N(rsp), rsp.ray_start_end_idx.shape[0]
        d = rgb_samples.device
        pred_rgb = torch.zeros(R, 3, device=d); pred_depth = torch.zeros(R, 1, device=d)
        bg = torch.zeros(R, 1, device=d); w = torch.zeros(N, 1, device=d)
        call("psdf_vr_volume_render_nerf", *rsp._rsp(), _f32(rgb_samples, "rgb", 3), _f32(radiance_samples, "radiance"),
             rsp.samples_z, rsp.samples_dt, pred_rgb, pred_depth, bg, w)
        return pred_rgb, pred_depth, bg, w

    @staticmethod
    def volume_render_nerf_backward(grad_pred_rgb, grad_bg_transmittance, grad_weight_per_sample, pred_rgb, rsp, rgb_samples,
                                    radiance_samples, ray_t_exit, use_ray_t_exit, bg_transmittance):
        N = rgb_samples.shape[0]
        d = rgb_samples.device
        g_rgb = torch.zeros(N, 3, device=d); g_rad = torch.zeros(N, 1, device=d)
        call("psdf_vr_volume_render_nerf_backward", *rsp._rsp(), _f32(grad_pred_rgb, "grad_pred_rgb"),
             _f32(grad_bg_transmittance, "grad_bg"), _f32(pred_rgb, "pred_rgb"), _f32(bg_transmittance, "bg_T"),
             _f32(rgb_samples, "rgb", 3), _f32(radiance_samples, "radiance"), rsp.samples_dt, g_rgb, g_rad)
        return g_rgb, g_rad


# ======================================================================================================
class PermutoSDF:
    """include/permuto_sdf/PermutoSDF.cuh:46-55 (static ops on the hot path; the rest are out of scope)"""

    @staticmethod
    def spherical_harmonics(dirs, degree):
        dr = _f32(dirs, "dirs", 3)
        degree = int(degree)
        if degree < 1 or degree > 7:
            raise RuntimeError("degree should be in 1..7")
        out = torch.empty(dr.shape[0], degree * degree, device=dr.device)
        call("psdf_spherical_harmonics", dr.shape[0], degree, dr, out)
        return out

    @staticmethod
    def random_rays_from_reel(tensor_reel, nr_rays):
        rgb = tensor_reel.rgb_reel
        nr_images, H, W = rgb.shape[0], rgb.shape[2], rgb.shape[3]
        d = rgb.device
        R = int(nr_rays)
        pix = torch.randint(0, H * W, (R,), dtype=torch.int32, device=d)
        img = torch.randint(0, nr_images, (R,), dtype=torch.int32, device=d)
        return PermutoSDF.rays_from_reel_indices(tensor_reel, pix, img)

    @staticmethod
    def rays_from_reel_indices(tensor_reel, pix, img):
        """same kernel as random_rays_from_reel with caller supplied (pixel, image) indices"""
        rgb = tensor_reel.rgb_reel
        mask = getattr(tensor_reel, "mask_reel", None)
        nr_images, H, W = rgb.shape[0], rgb.shape[2], rgb.shape[3]
        d = rgb.device
        R = pix.shape[0]
        has_mask = mask is not None and mask.numel() > 0
        o = torch.empty(R, 3, device=d); dr = torch.empty(R, 3, device=d)
        gt = torch.empty(R, 3, device=d); gm = torch.empty(R, 1, device=d)
        call("psdf_random_rays_from_reel", R, nr_images, H, W, _f32(rgb, "rgb_reel"), _f32(mask, "mask_reel") if has_mask else None,
             _f32(tensor_reel.K_reel, "K_reel"), _f32(tensor_reel.tf_world_cam_reel, "tf_world_cam_reel"), pix.contiguous(),
             img.contiguous(), 1 if has_mask else 0, o, dr, gt, gm)
        return o, dr, gt, gm, img

    @staticmethod
    def meshgrid3d(min_v, max_v, nr_points_per_dim):
        lin = torch.linspace(min_v, max_v, nr_points_per_dim, device=_dev())
        g = torch.meshgrid(lin, lin, lin, indexing="ij")
        return torch.stack(g, -1)


class TrainParams:
    """include/permuto_sdf/TrainParams.h:12-26 -- 4 booleans read from the cfg by the reference; plain holder here."""

    def __init__(self):
        self._v = dict(with_visdom=False, with_tensorboard=False, with_wandb=False, save_checkpoint=False)

    @staticmethod
    def create(cfg_path=None):
        return TrainParams()

    def with_visdom(self): return self._v["with_visdom"]
    def with_tensorboard(self): return self._v["with_tensorboard"]
    def with_wandb(self): return self._v["with_wandb"]
    def save_checkpoint(self): return self._v["save_checkpoint"]
    def set_with_visdom(self, v): self._v["with_visdom"] = bool(v)
    def set_with_tensorboard(self, v): self._v["with_tensorboard"] = bool(v)
    def set_with_wandb(self, v): self._v["with_wandb"] = bool(v)
    def set_save_checkpoint(self, v): self._v["save_checkpoint"] = bool(v)


class NGPGui:
    """include/permuto_sdf/NGPGui.h -- OpenGL viewer panel; not part of the hot path."""

    @staticmethod
    def create(view=None):
        raise RuntimeError("NGPGui needs the EasyPBR viewer; out of scope for the GPU hot path")


__all__ = ["PermutoSDF", "Sphere", "OccupancyGrid", "RaySamplesPacked", "VolumeRendering", "RaySampler", "TrainParams", "NGPGui"]
