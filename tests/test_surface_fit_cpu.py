"""Host logic of SurfaceFit: the refusals of the constructor and of step() (each with its reason), the autograd restatement of sdf_loss
against the reference's formula, and the checkpoint state. Nothing here needs a device: clouds that must fail before any device work are
CPU or meta tensors, and step() runs on an object built without models."""
import math

import pytest
import torch
import torch.nn.functional as F

from permuto_sdf_b200.surface_fit import SurfaceFit, _check_counts, sdf_loss


def _cloud(P=10, device="cpu"):
    return torch.zeros(P, 3, device=device), torch.zeros(P, 3, device=device)


@pytest.mark.parametrize("points, normals, reason", [
    (torch.zeros(10, 4), torch.zeros(10, 3), r"points should have shape \[P,3\]"),
    (torch.zeros(10, 3), torch.zeros(10), r"normals should have shape \[P,3\]"),
    (torch.zeros(10, 3, dtype=torch.float64), torch.zeros(10, 3), "points must be float32"),
    (torch.zeros(10, 3), torch.zeros(10, 3, dtype=torch.float16), "normals must be float32"),
    (torch.zeros(10, 3), torch.zeros(9, 3), "10 points but 9 normals"),
    (torch.zeros(10, 3), torch.zeros(10, 3, device="meta"), "points on cpu but normals on meta"),
    (torch.zeros(0, 3), torch.zeros(0, 3), "point cloud is empty"),
    (torch.empty(2 ** 30, 3, device="meta"), torch.empty(2 ** 30, 3, device="meta"), "32-bit row indexing"),
    (torch.zeros(10, 3), torch.zeros(10, 3), "must be on a CUDA device"),
    ([[0.0, 0.0, 0.0]], torch.zeros(1, 3), "points must be a tensor"),
])
def test_constructor_refusals(points, normals, reason):
    with pytest.raises(RuntimeError, match=reason):
        SurfaceFit(points, normals)


@pytest.mark.parametrize("ns, no, reason", [(0, 30000, "at least one surface and one box point"), (3000, 0, "at least one surface"),
                                            (-1, 5, "at least one"), (2 ** 29, 2 ** 29, "32-bit row indexing")])
def test_step_refusals(ns, no, reason):
    fit = SurfaceFit.__new__(SurfaceFit)          # no model: the counts are checked before anything runs
    with pytest.raises(RuntimeError, match=reason):
        fit.step(ns, no)
    with pytest.raises(RuntimeError, match=reason):
        fit.fit(3, ns, no)


def test_counts_at_the_limit():
    assert _check_counts(1, 1) == (1, 1)
    n = (2 ** 31 - 1) // 3
    assert _check_counts(1, n - 1) == (1, n - 1)


def test_sdf_loss_is_the_reference_formula():
    """sdf_utils.py:16-57 written out term by term, in fp64, with rows at sdf = 0, |g| = 0 and |g| = 1"""
    g = torch.Generator().manual_seed(3)
    Ns, No = 7, 11
    s_sdf, o_sdf = torch.randn(Ns, 1, generator=g, dtype=torch.float64), torch.randn(No, 1, generator=g, dtype=torch.float64) * 0.02
    s_g, o_g = torch.randn(Ns, 3, generator=g, dtype=torch.float64), torch.randn(No, 3, generator=g, dtype=torch.float64)
    nrm = torch.randn(Ns, 3, generator=g, dtype=torch.float64)
    s_sdf[0], o_sdf[0], s_g[1], s_g[2] = 0.0, 0.0, 0.0, torch.tensor([1.0, 0.0, 0.0], dtype=torch.float64)
    got = sdf_loss(s_sdf, s_g, o_sdf, o_g, nrm)
    eik = (torch.cat([s_g, o_g]).norm(dim=-1) - 1).abs().mean()
    cos = F.cosine_similarity(s_g, nrm, dim=-1)
    want = eik * 5e1 + (1 - cos).mean() * 1e2 + s_sdf.abs().mean() * 3e3 + torch.exp(-1e2 * o_sdf.abs()).mean() * 1e2
    assert math.isclose(float(got), float(want), rel_tol=1e-14)
    t = sdf_loss.terms
    assert math.isclose(float(t[0]), float(eik), rel_tol=1e-14) and math.isclose(float(t[2]), float(s_sdf.abs().mean()), rel_tol=1e-14)
    with pytest.raises(NotImplementedError):
        sdf_loss(s_sdf, s_g, o_sdf, o_g, nrm, eik_clamp=0.1)


def test_aabb_mirrors_the_reference_box():
    from permuto_sdf_b200 import AABB
    box = AABB([1.0, 2.0, 0.5], [0.1, 0.0, -0.2])
    assert box.max_bounds.tolist() == [0.5, 1.0, 0.25] and box.min_bounds.tolist() == [-0.5, -1.0, -0.25]
    p = torch.tensor([[0.1, 0.0, -0.2], [0.65, 0.0, -0.2], [0.55, 0.99, 0.04], [0.1, -1.0, -0.2]])
    assert box.check_point_inside_primitive(p).view(-1).tolist() == [True, False, True, False]
    with pytest.raises(RuntimeError, match="3 components"):
        AABB([1.0, 1.0], [0, 0, 0])
