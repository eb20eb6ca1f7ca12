"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Python front-end of oracle/_ref/libpsdf_ref_gpu.so: the UNMODIFIED reference CUDA kernels
(the original project's kernels/permuto_sdf/*GPU.cuh, compiled for sm_90a by oracle/ref_shim/Makefile) launched
the way the reference host code does (src/*.cu): grid ceil(n/256) x 256 threads, same output initial
values. Needs a GPU; used by the `-m gpu` parity tests, by tests/golden/make_ref_golden.py to produce
reference-made fixtures, and by bench.py to time the reference kernels next to ours.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libpsdf_ref_gpu.so")
_LIB = None
PCG_STATE = 0x853C49E6748FEA9B
PCG_INC = 0xDA3E39CB94B95BDB


def available():
    return os.path.exists(SO)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(SO)
    return _LIB


def _a(v):
    if v is None:
        return ctypes.c_void_p(0)
    if isinstance(v, torch.Tensor):
        assert v.is_cuda and v.is_contiguous(), "reference shim needs contiguous CUDA tensors"
        return ctypes.c_void_p(v.data_ptr())
    if isinstance(v, bool):
        return ctypes.c_bool(v)
    if isinstance(v, float):
        return ctypes.c_float(v)
    if isinstance(v, int):
        return ctypes.c_int(v)
    return v


def _call(name, *args):
    fn = getattr(lib(), name)
    fn.restype = ctypes.c_int
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = fn(*[_a(a) for a in args], st)
    if rc != 0:
        raise RuntimeError("%s -> cuda error %d" % (name, rc))


def U64(v):
    return ctypes.c_uint64(int(v))


def _e(*shape, dtype=torch.float32):
    return torch.empty(*shape, dtype=dtype, device="cuda")


def _z(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype, device="cuda")


class Packed:
    def __init__(self, R, M):
        self.pos, self.pos4, self.dirs = _e(M, 3), _z(M, 4), _e(M, 3)
        self.z, self.dt, self.sdf = _e(M, 1), _e(M, 1), _z(M, 1)
        self.fixed_dt = _e(R, 1)
        self.start_end = _e(R, 2, dtype=torch.int32)
        self.cur = _z(1, dtype=torch.int32)
        self.max_nr_samples = M
        self.equal, self.fixed_n, self.has_sdf = False, 0, False

    def rsp(self):
        return (self.start_end.shape[0], self.z.shape[0], self.max_nr_samples, self.start_end, bool(self.equal), int(self.fixed_n))

    def compact(self):
        R = self.start_end.shape[0]
        exact = int((self.start_end[:, 1] - self.start_end[:, 0]).sum().item())
        q = Packed(R, exact)
        q.equal, q.fixed_n, q.has_sdf = self.equal, self.fixed_n, self.has_sdf
        _call("ref_packed_compact", R, self.z.shape[0], exact, self.pos, self.pos4, self.dirs, self.z, self.dt, self.sdf, self.fixed_dt,
              self.start_end, q.pos, q.pos4, q.dirs, q.z, q.dt, q.sdf, q.fixed_dt, q.start_end, q.cur)
        return q


def tdev(v):
    return torch.tensor(list(v), dtype=torch.float32, device="cuda")


def sphere_ray_intersection(radius, center, o, d):
    n = o.shape[0]
    pe, te, px, tx, hit = _e(n, 3), _e(n, 1), _e(n, 3), _e(n, 1), _e(n, 1, dtype=torch.bool)
    _call("ref_sphere_ray_intersection", n, float(radius), tdev(center), o, d, pe, te, px, tx, hit)
    return pe, te, px, tx, hit


def sphere_rand_points_inside(radius, center, phi, ct, u):
    n = phi.shape[0]
    pts = _e(n, 3)
    _call("ref_sphere_rand_points_inside", n, float(radius), tdev(center), phi, ct, u, pts)
    return pts


def occ_grid_points(V, extent, trans, idx=None, randomize=False, state=PCG_STATE, inc=PCG_INC):
    if idx is None:
        n = V ** 3
        out = _e(n, 3)
        _call("ref_occ_compute_grid_points", n, V, float(extent), tdev(trans), U64(state), U64(inc), bool(randomize), out)
    else:
        n = idx.shape[0]
        out = _e(n, 3)
        _call("ref_occ_compute_random_sample_of_grid_points", n, V, float(extent), tdev(trans), idx, U64(state), U64(inc), bool(randomize), out)
    return out


def occ_update_with_density(V, density, idx, decay, thresh, values, occ):
    if idx is None:
        _call("ref_occ_update_with_density", V ** 3, density, V, float(decay), float(thresh), values, occ)
    else:
        _call("ref_occ_update_with_density_random_sample", idx.shape[0], density, V, idx, float(decay), float(thresh), values, occ)


def occ_update_with_sdf(V, extent, sdf, idx, inv_s, thresh, values, occ):
    if idx is None:
        _call("ref_occ_update_with_sdf", V ** 3, sdf, float(extent), V, float(inv_s), 1.0, float(thresh), values, occ)
    else:
        inv = torch.tensor([float(inv_s)], device="cuda")
        _call("ref_occ_update_with_sdf_random_sample", idx.shape[0], sdf, float(extent), V, idx, inv, float(thresh), values, occ)


def occ_check_occupancy(V, extent, trans, occ, pts):
    out = torch.ones(pts.shape[0], 1, dtype=torch.bool, device="cuda")
    _call("ref_occ_check_occupancy", pts.shape[0], V, float(extent), tdev(trans), occ, pts, out)
    return out


def occ_samples_in_occupied_regions(V, extent, trans, o, d, te, tx, occ, min_dist, max_per_ray, jitter=False, state=PCG_STATE,
                                    inc=PCG_INC, pool=2 * 1024 * 1024):
    R = o.shape[0]
    p = Packed(R, pool)
    _call("ref_occ_compute_samples_in_occupied_regions", R, V, float(extent), tdev(trans), o, d, te, tx, occ, float(min_dist),
          int(max_per_ray), pool, U64(state), U64(inc), bool(jitter), p.pos, p.dirs, p.z, p.dt, p.fixed_dt, p.start_end, p.cur)
    return p


def occ_first_sample_start(V, extent, trans, o, d, te, tx, occ, pool=2 * 1024 * 1024):
    R = o.shape[0]
    p = Packed(R, pool)
    _call("ref_occ_compute_first_sample_start_of_occupied_regions", R, V, float(extent), tdev(trans), o, d, te, tx, occ, pool, p.pos,
          p.dirs, p.z, p.dt, p.fixed_dt, p.start_end, p.cur)
    return p


def occ_advance_to_next_occupied(V, extent, trans, dirs, pos, occ):
    pos = pos.clone()
    within = torch.ones(pos.shape[0], 1, dtype=torch.bool, device="cuda")
    _call("ref_occ_advance_sample_to_next_occupied_voxel", pos.shape[0], V, float(extent), tdev(trans), dirs, pos, occ, within)
    return pos, within


def packed_per_sample_ray_idx(start_end, nr_samples):
    out = _z(nr_samples, dtype=torch.int32)
    _call("ref_packed_per_sample_ray_idx", start_end.shape[0], nr_samples, start_end, out)
    return out


def sampler_fg(o, d, te, tx, radius, center, min_dist, max_per_ray, jitter=False, state=PCG_STATE, inc=PCG_INC):
    R = o.shape[0]
    M = R * max_per_ray
    p = Packed(R, M)
    _call("ref_sampler_fg", R, o, d, te, tx, float(radius), tdev(center), float(min_dist), int(max_per_ray), M, U64(state), U64(inc),
          bool(jitter), p.pos, p.dirs, p.z, p.dt, p.fixed_dt, p.start_end, p.cur)
    return p


def sampler_bg(o, d, tx, n_per_ray, radius, center, randomize=False, contract=False, state=PCG_STATE, inc=PCG_INC):
    R = o.shape[0]
    p = Packed(R, R * n_per_ray)
    p.equal, p.fixed_n = True, n_per_ray
    _call("ref_sampler_bg", R, n_per_ray, o, d, tx, float(radius), tdev(center), U64(state), U64(inc), bool(randomize), bool(contract),
          p.pos, p.pos4, p.dirs, p.z, p.dt, p.fixed_dt, p.start_end)
    return p


def vr_cumprod(p, alpha):
    N, R = p.z.shape[0], p.start_end.shape[0]
    T, bg = _z(N, 1), torch.ones(R, 1, device="cuda")
    _call("ref_vr_cumprod_alpha2transmittance", *p.rsp(), alpha, T, bg)
    return T, bg


def vr_integrate(p, vals, w):
    out = _z(p.start_end.shape[0], 3)
    _call("ref_vr_integrate_with_weights", *p.rsp(), vals, w, out)
    return out


def vr_sdf2alpha(p, sdf, inv_s, dynamic, mult):
    alpha = _z(p.z.shape[0], 1)
    _call("ref_vr_sdf2alpha", *p.rsp(), p.fixed_dt, p.dt, sdf, float(inv_s), bool(dynamic), float(mult), alpha)
    return alpha


def vr_sum(p, vals):
    D = vals.shape[1]
    s_ray, s_smp = _z(p.start_end.shape[0], D), _z(p.z.shape[0], D)
    _call("ref_vr_sum_over_each_ray", *p.rsp(), D, vals, s_ray, s_smp)
    return s_ray, s_smp


def vr_cumsum(p, vals, inverse):
    out = _z(p.z.shape[0], 1)
    _call("ref_vr_cumsum_over_each_ray", *p.rsp(), vals, bool(inverse), out)
    return out


def vr_cdf(p, w):
    out = _z(p.z.shape[0], 1)
    _call("ref_vr_compute_cdf", *p.rsp(), w, out)
    return out


def vr_importance_sample(o, d, p, cdf, nr_imp, jitter=False, state=PCG_STATE, inc=PCG_INC):
    R = p.start_end.shape[0]
    q = Packed(R, R * nr_imp)
    q.equal, q.fixed_n = True, nr_imp
    _call("ref_vr_importance_sample", *p.rsp(), o, d, p.fixed_dt, p.z, cdf, nr_imp, U64(state), U64(inc), bool(jitter), q.pos, q.dirs, q.z,
          q.start_end)
    return q


def vr_combine(o, d, tx, p, q):
    R = p.start_end.shape[0]
    c_max = p.z.shape[0] + R * q.fixed_n
    c = Packed(R, c_max)
    c.has_sdf = p.has_sdf
    _call("ref_vr_combine_uniform_samples_with_imp", *p.rsp(), o, d, tx, p.fixed_dt, p.z, p.sdf, bool(p.has_sdf), q.fixed_n, q.z, q.sdf,
          bool(q.has_sdf), c_max, c.pos, c.dirs, c.z, c.dt, c.sdf, c.fixed_dt, c.start_end, c.cur)
    return c


def vr_cumprod_backward(p, gT, g_bg, alpha, T, bg_T, cumsumLV):
    g = _z(p.z.shape[0], 1)
    _call("ref_vr_cumprod_alpha2transmittance_backward", *p.rsp(), gT, g_bg, alpha, T, bg_T, cumsumLV, g)
    return g


def vr_integrate_backward(p, g_pred, vals, w, pred):
    N = p.z.shape[0]
    g_vals, g_w = _z(N, 3), _z(N, 1)
    _call("ref_vr_integrate_with_weights_backward", *p.rsp(), g_pred, vals, w, pred, g_vals, g_w)
    return g_vals, g_w


def vr_sum_backward(p, g_ray, g_sample, vals):
    g = torch.zeros_like(g_sample)
    _call("ref_vr_sum_over_each_ray_backward", *p.rsp(), g_sample.shape[1], g_ray, g_sample, vals, g)
    return g


def vr_compute_dt(p, tx, use_t_exit):
    dt = _z(p.z.shape[0], 1)
    _call("ref_vr_compute_dt", *p.rsp(), bool(use_t_exit), tx, p.z, dt)
    return dt


def vr_render_nerf(p, tx, rgb, radiance):
    N, R = p.z.shape[0], p.start_end.shape[0]
    pred, depth, bg, w = _z(R, 3), _z(R, 1), _z(R, 1), _z(N, 1)
    _call("ref_vr_volume_render_nerf", *p.rsp(), tx, rgb, radiance, p.z, p.dt, pred, depth, bg, w)
    return pred, depth, bg, w


def vr_render_nerf_backward(p, g_pred, g_bg, pred, tx, bg, rgb, radiance):
    N = p.z.shape[0]
    g_rgb, g_rad = _z(N, 3), _z(N, 1)
    _call("ref_vr_volume_render_nerf_backward", *p.rsp(), g_pred, g_bg, _z(N, 1), pred, tx, bg, rgb, radiance, p.dt, g_rgb, g_rad)
    return g_rgb, g_rad


def spherical_harmonics(dirs, degree):
    out = _e(dirs.shape[0], degree * degree)
    _call("ref_spherical_harmonics", dirs.shape[0], int(degree), dirs, out)
    return out


def random_rays_from_reel(rgb_reel, mask_reel, K, tf, pix, img):
    R = pix.shape[0]
    nimg, _, H, W = rgb_reel.shape
    o, d, gt, gm = _e(R, 3), _e(R, 3), _e(R, 3), _e(R, 1)
    has_mask = mask_reel is not None
    _call("ref_random_rays_from_reel", R, nimg, H, W, rgb_reel, mask_reel if has_mask else rgb_reel, K, tf, pix, img, bool(has_mask), o, d, gt, gm)
    return o, d, gt, gm
