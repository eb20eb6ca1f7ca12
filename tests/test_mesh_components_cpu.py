"""Connected components of a mesh without a GPU: the argument checks of Mesh.connected_components, remove_small_components and
keep_largest_component, the C ABI's new entry points and their limits, and a compile check that the kernels of csrc/mesh_components.cu
exist and do not spill."""
import ctypes
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from permuto_sdf_b200 import _lib
from permuto_sdf_b200.mesh import Mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENTRY_POINTS = ("psdf_mesh_components_workspace_bytes", "psdf_mesh_components", "psdf_mesh_components_keep")
KERNELS = ("k_cc_init", "k_cc_link", "k_cc_compress", "k_cc_count", "k_cc_roots", "k_cc_keep")


def tri_mesh(faces=None, dtype=torch.int32):
    F = torch.tensor([[0, 1, 2]] if faces is None else faces, dtype=dtype)
    return Mesh(torch.zeros(3, 3), F)


def all_calls(m):
    return [m.connected_components, lambda: m.remove_small_components(1), m.keep_largest_component]


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("dtype", [torch.int64, torch.float32, torch.uint8])
def test_faces_of_another_dtype_are_refused(dtype):
    for fn in all_calls(tri_mesh(dtype=dtype)):
        with pytest.raises(RuntimeError, match="int32"):
            fn()


@pytest.mark.parametrize("F", [torch.zeros(6, dtype=torch.int32), torch.zeros(2, 4, dtype=torch.int32),
                               torch.zeros(1, 3, 1, dtype=torch.int32)])
def test_faces_of_another_shape_are_refused(F):
    for fn in all_calls(Mesh(torch.zeros(3, 3), F)):
        with pytest.raises(RuntimeError, match=r"shape \[F,3\]"):
            fn()


def test_faces_that_are_not_a_tensor_are_refused():
    for fn in all_calls(Mesh(torch.zeros(3, 3), np.array([[0, 1, 2]], dtype=np.int32))):
        with pytest.raises(RuntimeError, match="int32 tensor"):
            fn()


def test_cpu_tensors_are_refused():
    for fn in all_calls(tri_mesh()):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn()


@pytest.mark.parametrize("k", [-1, -(2 ** 40), 1.0, 2.5, "3", None, True, np.float32(4)])
def test_min_faces_must_be_a_non_negative_integer(k):
    with pytest.raises(RuntimeError, match="min_faces"):
        tri_mesh().remove_small_components(k)


# ------------------------------------------------------------------------------------------------ C ABI
def test_abi_declares_and_exports_the_entry_points():
    syms = _lib.declared_symbols()
    assert set(ENTRY_POINTS) <= set(syms)
    ret, args = _lib.PROTOS["psdf_mesh_components_keep"]
    assert ret == "int" and [a for a, _ in args] == ["V", "largest", "min_faces", "workspace", "keep", "stream"]
    assert dict(args)["min_faces"] == "long long"
    assert _lib.PROTOS["psdf_mesh_components_workspace_bytes"][0] == "long long"
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRY_POINTS:
        assert hasattr(lib, s), "library does not export " + s


def test_workspace_size_and_limits():
    lib = _lib.load_library()
    ws = lib.psdf_mesh_components_workspace_bytes
    assert ws(0, 0) == 256 and ws(5, 7) == 256 + 40 and ws(2 ** 31 - 1, 2 ** 31 - 1) == 256 + 8 * (2 ** 31 - 1)
    assert ws(2 ** 31, 1) == -3 and ws(1, 2 ** 31) == -3
    assert ws(-1, 0) == -1 and ws(0, -1) == -1


def test_argument_errors_before_any_launch():
    lib = _lib.load_library()
    assert lib.psdf_mesh_components(-1, 0, None, None, None) == -1
    assert lib.psdf_mesh_components(3, 1, None, 8, None) == -1           # faces missing
    assert lib.psdf_mesh_components_keep(3, 0, -1, 8, 8, None) == -1    # negative min_faces
    assert lib.psdf_mesh_components_keep(3, 0, 0, None, 8, None) == -1
    assert lib.psdf_mesh_components_keep(0, 1, 0, 8, None, None) == 0    # nothing to do


# ------------------------------------------------------------------------------------------------ compile check
@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("mesh_components.cu",))}


def test_kernels_are_built_and_do_not_spill(kernels):
    cc = {k: r for k, r in kernels.items() if k.startswith("k_cc_")}
    assert set(cc) == set(KERNELS)
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in cc.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling
