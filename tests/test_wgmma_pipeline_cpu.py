"""ptxas keeps the wgmma chains of the hot fused kernels pipelined (tools/wgmma_report.py; needs nvcc, no GPU).

A chain that ptxas serializes waits for every HGMMA on its own (C7514 / C7515 / C7520); a batched chain issues a k-loop's three split
products, over all streams, behind one WARPGROUP.DEPBAR."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

SERIALIZED = ("C7514", "C7515", "C7520")
# kernels on the training / tracing paths whose chains this project keeps batched
PIPELINED = ["k_sdf_fused_dual<3>", "k_sdf_fused_dual<4>", "k_sdf_fused_backward<3>", "k_sdf_fused_backward<4>", "k_rgb_fused_backward",
             "k_sdf_sphere_trace<3, false>", "k_sdf_sphere_trace<3, true>", "k_sdf_sphere_trace<4, false>", "k_sdf_sphere_trace<4, true>"]
# value-only and colour-forward kernels that were batched before the kernels above
ALREADY_BATCHED = ["k_sdf_fused<false, 3>", "k_sdf_fused<false, 4>", "k_sdf_fused<true, 3>", "k_rgb_fused"]


@pytest.fixture(scope="module")
def report():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    rows = wgmma_report.report(("fused_sdf.cu", "fused_sdf_bwd.cu", "fused_rgb.cu", "fused_rgb_bwd.cu"))
    return {r["kernel"]: r for r in rows}


@pytest.mark.parametrize("kernel", PIPELINED + ALREADY_BATCHED)
def test_wgmma_chains_not_serialized(report, kernel):
    r = report[kernel]
    assert r["hgmma"] > 0
    assert not [c for c in SERIALIZED if c in r["diag"]], r["diag"]
    assert 3 * r["depbar"] <= r["hgmma"], "%d WARPGROUP.DEPBAR for %d HGMMA" % (r["depbar"], r["hgmma"])
