"""Camera rigs and an in-memory reel, so that any mesh becomes a multi-view training scene whose answer is known: cameras from look_at,
sphere_cameras or orbit_cameras, images from Mesh.render, and TensorReel holding them in the layout the trainers and metrics read."""
import math

import torch

from .mesh import fibonacci_directions


def look_at(eyes, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    """camera-to-world transforms of cameras at eyes [I,3] looking at target -> tf_world_cam float32 [I,4,4] on the eyes' device:
    z = normalize(target - eye), x = normalize(cross(up, z)), y = cross(z, x), in fp32 torch; the columns are x, y, z and the eye, the last
    row (0, 0, 0, 1). This is bench.analytic_reel's construction: given its eyes it gives its tf. An eye at the target, or one whose z is
    parallel to up, is refused."""
    e = torch.as_tensor(eyes, dtype=torch.float32)
    if e.dim() != 2 or e.shape[1] != 3:
        raise RuntimeError("look_at: eyes must have shape [I,3], got %s" % list(e.shape))
    if not bool(torch.isfinite(e).all()):
        raise RuntimeError("look_at: eyes has values that are not finite")
    tgt = torch.as_tensor(target, dtype=torch.float32, device=e.device)
    u = torch.as_tensor(up, dtype=torch.float32, device=e.device)
    if tgt.shape != (3,) or u.shape != (3,):
        raise RuntimeError("look_at: target and up must be 3-vectors")
    z = tgt - e
    zn = z.norm(dim=1, keepdim=True)
    if bool((zn == 0).any()):
        raise RuntimeError("look_at: eye %d is at the target" % int(torch.nonzero(zn[:, 0] == 0)[0]))
    z = z / zn
    x = torch.linalg.cross(u.expand_as(z), z)
    xn = x.norm(dim=1, keepdim=True)
    flat = xn[:, 0] <= 1e-6 * u.norm()
    if bool(flat.any()):
        raise RuntimeError("look_at: eye %d looks along up %s; its x axis is undefined" % (int(torch.nonzero(flat)[0]), u.tolist()))
    x = x / xn
    y = torch.linalg.cross(z, x)
    tf = torch.zeros(e.shape[0], 4, 4, dtype=torch.float32, device=e.device)
    tf[:, :3, 0], tf[:, :3, 1], tf[:, :3, 2], tf[:, :3, 3] = x, y, z, e
    tf[:, 3, 3] = 1.0
    return tf


def _intrinsics(nr_images, H, W, focal, device="cuda"):
    """K float32 [I,3,3] = [[f, 0, W/2], [0, f, H/2], [0, 0, 1]] for every image"""
    K = torch.tensor([[focal, 0.0, W / 2.0], [0.0, focal, H / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    return K.expand(int(nr_images), 3, 3).contiguous().to(device)


def _check_rig(fn, nr_images, H, W, focal, radius):
    if isinstance(nr_images, bool) or not isinstance(nr_images, int) or nr_images < 1:
        raise RuntimeError("%s: nr_images must be a positive integer, got %r" % (fn, nr_images))
    for name, v in (("H", H), ("W", W)):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise RuntimeError("%s: %s must be a positive integer, got %r" % (fn, name, v))
    for name, v in (("focal", focal), ("radius", radius)):
        if not (math.isfinite(float(v)) and float(v) > 0):
            raise RuntimeError("%s: %s must be positive and finite, got %r" % (fn, name, v))


def sphere_cameras(nr_images, H, W, focal, radius=1.2, target=(0.0, 0.0, 0.0), device="cuda"):
    """nr_images cameras at target + radius * fibonacci_directions(nr_images) (the directions of Mesh.ambient_occlusion), looking at
    target with up = +y -> (K float32 [I,3,3] of focal length `focal` and principal point (W/2, H/2), tf_world_cam float32 [I,4,4]) on
    `device`. bench.analytic_reel puts its cameras on the same radius-1.2 sphere, at random directions."""
    _check_rig("sphere_cameras", nr_images, H, W, focal, radius)
    eyes = torch.from_numpy(fibonacci_directions(nr_images)) * float(radius) + torch.as_tensor(target, dtype=torch.float32)
    return _intrinsics(nr_images, H, W, focal, device), look_at(eyes.to(device), target)


def orbit_cameras(nr_images, H, W, focal, radius=1.8, elevation_deg=30.0, target=(0.0, 0.0, 0.0), device="cuda"):
    """the orbit of render_orbit.py: nr_images cameras at distance `radius` from target, `elevation_deg` above its xz plane, evenly spaced
    in azimuth about +y starting on +z (eye k at azimuth a = 2 pi k / nr_images: target + radius (cos e sin a, sin e, cos e cos a)), looking
    at target with up = +y -> (K [I,3,3], tf_world_cam [I,4,4]) as sphere_cameras"""
    _check_rig("orbit_cameras", nr_images, H, W, focal, radius)
    if not abs(float(elevation_deg)) < 90:
        raise RuntimeError("orbit_cameras: elevation_deg must lie strictly between -90 and 90, got %r" % (elevation_deg,))
    a = torch.arange(nr_images, dtype=torch.float64) * (2 * math.pi / nr_images)
    el = math.radians(float(elevation_deg))
    dirs = torch.stack([math.cos(el) * torch.sin(a), torch.full_like(a, math.sin(el)), math.cos(el) * torch.cos(a)], 1)
    eyes = (dirs * float(radius)).float() + torch.as_tensor(target, dtype=torch.float32)
    return _intrinsics(nr_images, H, W, focal, device), look_at(eyes.to(device), target)


class TensorReel:
    """a reel of I images held in tensors, with the attributes the trainers (step_from_reel, evaluate, render_frame) and metrics read:
    rgb_reel float32 [I,3,H,W] (already multiplied by the mask), mask_reel float32 [I,1,H,W] or None (no masks), K_reel float32 [I,3,3],
    tf_world_cam_reel float32 [I,4,4] (camera to world, row-major). Every tensor must be contiguous and on one device (the trainers need
    CUDA); dtype, shape, device and contiguity are checked here, once, so that a mis-shaped reel fails at construction rather than inside
    a kernel."""

    def __init__(self, rgb, mask, K, tf_world_cam):
        fn = "TensorReel"
        if not isinstance(rgb, torch.Tensor) or rgb.dim() != 4 or rgb.shape[1] != 3:
            raise RuntimeError("%s: rgb must be a tensor of shape [I,3,H,W], got %s" % (fn, _shape(rgb)))
        I, _, H, W = rgb.shape
        if I < 1 or H < 1 or W < 1:
            raise RuntimeError("%s: rgb has shape %s; a reel needs at least one image of at least one pixel" % (fn, list(rgb.shape)))
        if H * W > 2 ** 31 - 1:
            raise RuntimeError("%s: a %d x %d image has more pixels than the ray kernel indexes in 32 bits" % (fn, H, W))
        expect = {"rgb": (I, 3, H, W), "mask": (I, 1, H, W), "K": (I, 3, 3), "tf_world_cam": (I, 4, 4)}
        for name, x in (("rgb", rgb), ("mask", mask), ("K", K), ("tf_world_cam", tf_world_cam)):
            if x is None and name == "mask":
                continue
            if not isinstance(x, torch.Tensor) or tuple(x.shape) != expect[name]:
                raise RuntimeError("%s: %s must be a tensor of shape %s, got %s" % (fn, name, list(expect[name]), _shape(x)))
            if x.dtype != torch.float32:
                raise RuntimeError("%s: %s must be float32, got %s" % (fn, name, x.dtype))
            if x.device != rgb.device:
                raise RuntimeError("%s: %s must be on rgb's device %s, got %s" % (fn, name, rgb.device, x.device))
            if not x.is_contiguous():
                raise RuntimeError("%s: %s must be contiguous" % (fn, name))
        self.rgb_reel, self.mask_reel, self.K_reel, self.tf_world_cam_reel = rgb, mask, K, tf_world_cam


def _shape(x):
    return list(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
