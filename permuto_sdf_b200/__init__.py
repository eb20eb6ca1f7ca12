"""permuto_sdf_b200 -- H100-native (sm_90a) implementation of PermutoSDF's per-ray training and
sphere-tracing hot path behind the reference's own Python operator API.

    permuto_sdf_b200.permuto_sdf              mirror of the pybind module `permuto_sdf` (src/PyBridge.cxx)
    permuto_sdf_b200.permutohedral_encoding   mirror of the external `permutohedral_encoding` package
    compat/                                   top-level `permuto_sdf` / `permutohedral_encoding` shims so the
                                              reference's permuto_sdf_py runs unchanged (see INTEGRATION.md)
    permuto_sdf_b200.patch_reference_models   routes the reference's own SDF / RGB classes through the fused tensor-core kernels
    permuto_sdf_b200.SurfaceFit / AABB        SDF from an oriented point cloud (train_sdf_from_mesh.py) on the fused kernels
    permuto_sdf_b200.SpaceTimeFit             space-time SDF from a point sequence (train_4d_sdf.py) on the fused kernels
    permuto_sdf_b200.NerfTrainer              NeRF training (train_nerf.py) on the fused kernels

All device work goes through the C ABI in include/psdf_b200.h (libpsdf_b200.so, hand-written CUDA).
There is no CPU or PyTorch fallback: importing is cheap, but any op raises if the library is missing
or the tensors are not on a CUDA device.
"""
from ._lib import LIB_PATH, call, declared_symbols, load_library  # noqa: F401
from .patch import patch_reference_models, unpatch_reference_models  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    # imported on first use, so that importing the package stays cheap (no torch import)
    if name == "SurfaceFit":
        from .surface_fit import SurfaceFit
        return SurfaceFit
    if name == "SpaceTimeFit":
        from .surface_fit import SpaceTimeFit
        return SpaceTimeFit
    if name == "NerfTrainer":
        from .nerf_train import NerfTrainer
        return NerfTrainer
    if name == "AABB":
        from .permuto_sdf import AABB
        return AABB
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
