"""The reference-Python fixture (tests/golden/refpy_golden.npz + refpy_golden_bg.npz) is reproducible: where a checkout of the original
project is present (PERMUTO_SDF_REFERENCE, else its default location) the committed generator, run again, must give the committed arrays,
and the graft works on the original classes. Also checks the fixture's internal consistency everywhere."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIX = os.path.join(HERE, "golden", "refpy_golden.npz")
REF_PY = os.path.join(os.environ.get("PERMUTO_SDF_REFERENCE") or "/root/reference", "permuto_sdf_py")
NO_REF = "needs a checkout of the original project (PERMUTO_SDF_REFERENCE or its default location)"


def load_fixture(path):
    """the fixture and its background-model part (<name>_bg.npz) as one dict"""
    g = dict(np.load(path))
    g.update(np.load(path[:-len(".npz")] + "_bg.npz"))
    return g


def test_fixture_is_complete():
    G = load_fixture(FIX)
    keys = set(G.keys())
    for need in ("sdf_out.sdf", "sdf_grad.lattice_rows", "curv_out.curvature", "rgb_out.rgb", "rgb_grad.mlp.lipshitz_bound_per_layer.0",
                 "rgb_grad.cal.weight_delta", "bg_out.density", "neus_free.weights", "neus_forced.g_sdf", "imp_out.samples_z", "trace_out.points"):
        assert need in keys, need
    # the reference's state_dict key names travel with the fixture (checkpoint interoperability, SURVEY.md 8(f) rank 4)
    assert {"rgb.mlp.weights_per_layer.0", "rgb.mlp.biases_per_layer.3", "rgb.mlp.layers.2.weight", "rgb.mlp.lipshitz_bound_per_layer.1",
            "rgb.volume_renderer_neus.deviation_network.variance", "sdf.mlp_sdf.6.bias", "sdf.encoding.random_shift_per_level"} <= keys
    se = G["rgb_in.ray_start_end_idx"]
    assert (se[:, 1] >= se[:, 0]).all() and (se[3, 1] == se[3, 0]) and se[-1, 1] == G["rgb_in.points"].shape[0]
    # the Lipschitz clamp is active in the fixture: softplus(c) below at least one row sum of |W| in a layer
    for l in range(4):
        w, c = G["rgb.mlp.layers.%d.weight" % l], float(G["rgb.mlp.lipshitz_bound_per_layer.%d" % l][0])
        if np.log1p(np.exp(c)) < np.abs(w).sum(1).max():
            break
    else:
        pytest.fail("no active Lipschitz clamp in the fixture")


@pytest.mark.skipif(not os.path.isdir(REF_PY), reason=NO_REF)
def test_fixture_regenerates_from_the_reference(tmp_path):
    env = dict(os.environ, REFPY_GOLDEN_OUT=str(tmp_path / "again.npz"))
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_refpy_golden.py")], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    a, b = load_fixture(FIX), load_fixture(str(tmp_path / "again.npz"))
    assert set(a.keys()) == set(b.keys())
    for k in a.keys():
        if a[k].dtype.kind == "f":
            assert np.allclose(a[k], b[k], rtol=1e-5, atol=1e-7), k
        else:
            assert np.array_equal(a[k], b[k]), k


_PATCH_CHECK = r"""
import sys, torch
sys.path.insert(0, %r)
from oracle import refpy
M = refpy.install()
import permuto_sdf as ps
import permuto_sdf_b200
torch.manual_seed(0)
sdf = M.SDF(in_channels=3, boundary_primitive=ps.Sphere(0.5, [0, 0, 0]), geom_feat_size_out=32, nr_iters_for_c2f=10000)
with torch.no_grad():
    sdf.encoding.lattice_values.uniform_(-0.3, 0.3)
pts = (torch.rand(64, 3) - 0.5) * 0.8
a = sdf.get_sdf_and_gradient(pts.clone(), 3000)
orig_forward = M.SDF.forward
permuto_sdf_b200.patch_reference_models(M)
assert M.SDF.forward is not orig_forward and hasattr(M.SDF, "enable_fused_training") and hasattr(M.RGB, "enable_fused")
b = sdf.get_sdf_and_gradient(pts.clone(), 3000)           # CPU tensors: the grafted methods take the per-op branch (no fused path on CPU)
assert sdf.fused is None
for x, y in zip(a, b):
    assert torch.allclose(x, y, rtol=1e-6, atol=1e-7)
assert list(sdf.state_dict().keys()) == ["encoding.lattice_values", "encoding.random_shift_per_level"] + ["mlp_sdf.%%d.%%s" %% (i, n) for i in (0, 2, 4, 6) for n in ("weight", "bias")]
permuto_sdf_b200.unpatch_reference_models(M)
assert M.SDF.forward is orig_forward
print("PATCH-OK")
"""


@pytest.mark.skipif(not os.path.isdir(REF_PY), reason=NO_REF)
def test_patch_grafts_onto_the_real_reference_classes():
    """permuto_sdf_b200.patch_reference_models on the UNMODIFIED permuto_sdf_py/models/models.py (own process: oracle/refpy.py replaces
    sys.modules entries): methods replaced, instances keep parameters / state_dict keys / results, unpatch restores"""
    r = subprocess.run([sys.executable, "-c", _PATCH_CHECK % ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "PATCH-OK" in r.stdout, r.stderr[-3000:]
