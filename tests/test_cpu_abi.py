"""CPU-side checks of the drop-in boundary: the C-ABI library builds/loads without a GPU, exports every symbol
declared in include/psdf_b200.h, and the product path refuses to run without CUDA (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

from permuto_sdf_b200 import _lib


def test_header_parses_and_library_exports_every_symbol():
    syms = _lib.declared_symbols()
    assert len(syms) >= 35
    hdr = open(_lib.HEADER).read()
    # every psdf_ function named in the header text is covered by the parser
    names = set(re.findall(r"\b(psdf_[a-z0-9_]+)\s*\(", hdr))
    assert names == set(syms)
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(lib, s), "library does not export " + s


def test_library_identifies_itself():
    lib = _lib.load_library()
    assert lib.psdf_abi_version() == 2
    if not torch.cuda.is_available():
        assert lib.psdf_device_ok() == 0


def test_no_cpu_fallback():
    from permuto_sdf_b200 import call
    with pytest.raises(RuntimeError):
        call("psdf_spherical_harmonics", 4, 3, torch.zeros(4, 3), torch.zeros(4, 9))   # CPU tensors are rejected
    import permutohedral_encoding as pe
    if not torch.cuda.is_available():
        enc = pe.PermutoEncoding(3, 1024, 2, 2, [1.0, 0.1])
        with pytest.raises(RuntimeError):
            enc(torch.rand(5, 3))


def test_product_never_imports_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for dp, _, files in os.walk(os.path.join(root, "permuto_sdf_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")) and f != "smoke_test.py":
                txt = open(os.path.join(dp, f)).read()
                assert "oracle" not in txt.replace("oracle/", "").replace("the oracle", "").replace("against the oracle", "") or \
                    "import oracle" not in txt and "from oracle" not in txt, f
                assert "from oracle" not in txt and "import oracle" not in txt, "product file imports the oracle: " + f


def test_compat_names_match_reference_api():
    import permuto_sdf
    import permutohedral_encoding
    for n in ["PermutoSDF", "Sphere", "OccupancyGrid", "RaySamplesPacked", "VolumeRendering", "RaySampler", "TrainParams", "NGPGui"]:
        assert hasattr(permuto_sdf, n)
    vr = permuto_sdf.VolumeRendering
    for m in ["volume_render_nerf", "compute_dt", "cumprod_alpha2transmittance", "integrate_with_weights", "sdf2alpha", "sum_over_each_ray",
              "cumsum_over_each_ray", "compute_cdf", "importance_sample", "combine_uniform_samples_with_imp", "volume_render_nerf_backward",
              "cumprod_alpha2transmittance_backward", "integrate_with_weights_backward", "sum_over_each_ray_backward"]:
        assert callable(getattr(vr, m)), m          # src/PyBridge.cxx:105-122
    og = permuto_sdf.OccupancyGrid
    for m in ["make_grid_values", "make_grid_occupancy", "get_grid_values", "set_grid_values", "get_grid_occupancy", "set_grid_occupancy",
              "get_nr_voxels", "get_nr_voxels_per_dim", "compute_grid_points", "compute_random_sample_of_grid_points", "check_occupancy",
              "update_with_density", "update_with_density_random_sample", "update_with_sdf", "update_with_sdf_random_sample",
              "compute_samples_in_occupied_regions", "compute_first_sample_start_of_occupied_regions",
              "advance_sample_to_next_occupied_voxel"]:
        assert hasattr(og, m), m                     # src/PyBridge.cxx:60-81
    for m in ["compact_to_valid_samples", "compute_exact_nr_samples", "initialize_with_one_sample_per_ray", "set_sdf", "remove_sdf",
              "compute_per_sample_ray_idx"]:
        assert hasattr(permuto_sdf.RaySamplesPacked, m), m
    assert hasattr(permutohedral_encoding, "PermutoEncoding") and hasattr(permutohedral_encoding, "Coarse2Fine")
