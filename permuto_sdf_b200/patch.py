"""Make the fused tensor-core path reachable from the REFERENCE's own model classes.

Over compat/ the unmodified permuto_sdf_py/models/models.py runs on the per-op kernels (encoding kernels + torch.nn.Linear +
autograd). `patch_reference_models(M)` grafts the methods of this package's SDF / RGB onto the reference classes of the imported
module M, so that instances created by the reference's own code (`model_sdf = SDF(...)` in train_permuto_sdf.py:276-277) evaluate
through csrc/fused_sdf*.cu / fused_rgb*.cu:

    import permuto_sdf_py.models.models as M          # the reference, with <repo>/compat in front of sys.path
    import permuto_sdf_b200
    permuto_sdf_b200.patch_reference_models(M)
    model_sdf = M.SDF(in_channels=3, boundary_primitive=aabb, geom_feat_size_out=32, nr_iters_for_c2f=10000).to("cuda")
    model_sdf.enable_fused_training()                 # or let the first CUDA call do it: M.SDF.fused_auto = True

The classes keep their parameters, state_dict keys and constructor; only forward / get_sdf_and_gradient (SDF, models.py:176-259)
and forward (RGB, models.py:359-391) change, to the versions of permuto_sdf_b200/models.py (same results to ~1e-5, tests:
tests/test_refpy_golden_gpu.py against the reference's own outputs, tests/test_patch_gpu.py for the graft).
Shapes the fused kernels do not cover raise (no silent fall-back); `unpatch_reference_models(M)` restores the originals."""
import sys

_SDF_METHODS = ("window", "enable_fused_inference", "enable_fused_training", "forward", "get_sdf_and_gradient", "curvature_loss")
_RGB_METHODS = ("forward", "enable_fused", "_head")
_SAVED = {}


def patch_reference_models(M, auto_enable=True):
    """M: a module holding reference-shaped classes `SDF` and `RGB` (attributes encoding / mlp_sdf / c2f / nr_iters_for_c2f /
    geom_feat_size_out, resp. encoding / mlp (LipshitzMLP) / c2f / volume_renderer_neus). auto_enable: instances switch their fused
    path on at the first evaluation on CUDA tensors (otherwise call enable_fused_training() / enable_fused() yourself)."""
    from . import models as ours
    if id(M) in _SAVED:
        return M
    saved = {"SDF": {k: M.SDF.__dict__.get(k) for k in _SDF_METHODS + ("fused", "fused_training")},
             "RGB": {k: M.RGB.__dict__.get(k) for k in _RGB_METHODS + ("fused", "fused_head")}}
    for k in _SDF_METHODS:
        setattr(M.SDF, k, ours.SDF.__dict__[k])
    for k in _RGB_METHODS:
        setattr(M.RGB, k, ours.RGB.__dict__[k])
    M.SDF.fused, M.SDF.fused_training = None, False
    M.RGB.fused, M.RGB.fused_head = None, True
    if auto_enable:
        sdf_fwd, sdf_gsg, rgb_fwd = ours.SDF.forward, ours.SDF.get_sdf_and_gradient, ours.RGB.forward

        def _auto_sdf(self, points):
            if self.fused is None and points.is_cuda:
                self.enable_fused_training()

        def forward(self, points, iter_nr):
            _auto_sdf(self, points)
            return sdf_fwd(self, points, iter_nr)

        def get_sdf_and_gradient(self, points, iter_nr, method="autograd"):
            _auto_sdf(self, points)
            return sdf_gsg(self, points, iter_nr, method)

        def rgb_forward(self, points, *a, **k):
            if self.fused is None and points.is_cuda:
                self.enable_fused()
            return rgb_fwd(self, points, *a, **k)
        M.SDF.forward, M.SDF.get_sdf_and_gradient, M.RGB.forward = forward, get_sdf_and_gradient, rgb_forward
    _SAVED[id(M)] = saved
    return M


def unpatch_reference_models(M):
    saved = _SAVED.pop(id(M), None)
    if saved is None:
        return M
    for cls_name, d in saved.items():
        cls = getattr(M, cls_name)
        for k, v in d.items():
            if v is None:
                if k in cls.__dict__:
                    delattr(cls, k)
            else:
                setattr(cls, k, v)
    return M
