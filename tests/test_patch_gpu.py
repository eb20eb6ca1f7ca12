"""permuto_sdf_b200.patch_reference_models: reference-shaped classes (tests/refshape_models.py: the layout and formulas of
permuto_sdf_py/models/models.py, per-op kernels + autograd) evaluate through the fused tensor-core kernels after the graft, with the same
values and parameter gradients; unpatch restores the per-op path."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def test_reference_shaped_classes_run_fused_after_patch(cuda):
    import permuto_sdf_b200
    from permuto_sdf import Sphere
    import refshape_models as R
    M = types.ModuleType("refshape_copy")
    M.SDF, M.RGB = type("SDF", (R.SDF,), {}), type("RGB", (R.RGB,), {})
    torch.manual_seed(0)
    sph = Sphere(0.5, [0, 0, 0])
    sdf_m = M.SDF(3, sph, 32, 10000, nr_levels=16, capacity=2 ** 14).cuda()
    rgb_m = M.RGB(3, sph, 32, 1, nr_levels=16, capacity=2 ** 14).cuda()
    with torch.no_grad():
        for m in (sdf_m, rgb_m):
            m.encoding.lattice_values.uniform_(-0.3, 0.3)
    N = 3000
    pts = (torch.rand(N, 3, device="cuda") - 0.5) * 0.8
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, device="cuda"), dim=-1)
    ca, cb, cc = torch.randn(N, 1, device="cuda"), torch.randn(N, 3, device="cuda"), torch.randn(N, 3, device="cuda")

    def run():
        for m in (sdf_m, rgb_m):
            m.zero_grad()
        sdf, g, geom = sdf_m.get_sdf_and_gradient(pts.clone(), 5000)
        rgb = rgb_m(pts, dirs, g, geom, 5000)
        ((sdf * ca).sum() + (g * cb).sum() + (rgb * cc).sum()).backward()
        grads = [p.grad.detach().clone() for m in (sdf_m, rgb_m) for p in m.parameters() if p.grad is not None]
        return sdf.detach(), g.detach(), rgb.detach(), grads
    ref = run()                                                   # per-op kernels + autograd (what compat/ gives the reference)
    assert getattr(sdf_m, "fused", None) is None
    permuto_sdf_b200.patch_reference_models(M)
    got = run()                                                   # same instances, now through csrc/fused_sdf*.cu / fused_rgb*.cu
    assert sdf_m.fused is not None and sdf_m.fused_training and rgb_m.fused is not None
    for a, b in zip(got[:3], ref[:3]):
        assert rel(a, b) < 1e-3
    assert len(got[3]) == len(ref[3])
    for a, b in zip(got[3], ref[3]):
        assert rel(a, b) < 1e-3
    assert set(sdf_m.state_dict()) == {"encoding.lattice_values", "encoding.random_shift_per_level"} | {"mlp_sdf.%d.%s" % (i, n) for i in (0, 2, 4, 6) for n in ("weight", "bias")}
    permuto_sdf_b200.unpatch_reference_models(M)
    assert M.SDF.forward is R.SDF.forward or "forward" not in M.SDF.__dict__
