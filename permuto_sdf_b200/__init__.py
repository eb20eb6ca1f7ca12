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
    permuto_sdf_b200.extract_mesh_from_sdf_model / marching_cubes / Mesh   meshes from a trained SDF or a volume on the GPU
    permuto_sdf_b200.extract_mesh_from_density_model   meshes from a trained NeRF's density (NerfTrainer.model) on the GPU
    permuto_sdf_b200.load_mesh_sequence       the [P,4] point sequence of train_4d_sdf.py from a folder of meshes (ray-cast AO on the GPU)
    permuto_sdf_b200.mesh_distance            accuracy, completeness, chamfer and Hausdorff distance of two meshes (BVH queries on the GPU)
    permuto_sdf_b200.look_at / sphere_cameras / orbit_cameras / TensorReel   camera rigs and an in-memory reel; with Mesh.render
                                              (first hits on the GPU BVH) any mesh becomes a training scene
    permuto_sdf_b200.psnr / ssim              image metrics of evaluate_psnr.py on the GPU (metrics.py; Trainer.evaluate scores frames)

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
    if name in ("Mesh", "marching_cubes", "extract_mesh_from_sdf_model", "extract_mesh_from_density_model", "load_mesh_sequence",
                "mesh_distance"):
        from . import mesh
        return getattr(mesh, name)
    if name in ("look_at", "sphere_cameras", "orbit_cameras", "TensorReel"):
        from . import cameras
        return getattr(cameras, name)
    if name in ("psnr", "ssim"):
        from . import metrics
        return getattr(metrics, name)
    if name == "AABB":
        from .permuto_sdf import AABB
        return AABB
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
