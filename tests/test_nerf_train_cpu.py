"""NerfTrainer without a GPU: the refusals, the mirror of train_nerf.py's hyperparameters and losses, and the fp64 oracle of the
NerfHash kernels at D = 3 (the foreground network): error scales propagated and tangents equal to fp64 autograd."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import backward_fp64 as R


def test_hyperparameters_mirror_train_nerf():
    from permuto_sdf_b200.nerf_train import MASK_WEIGHT, OCC_DECAY, OCC_EVERY, OCC_NR_POINTS, OCC_THRESH, NerfHyperParams
    hp = NerfHyperParams()
    assert (hp.lr, hp.nr_rays, hp.max_nr_samples_per_ray, hp.min_dist_between_samples, hp.nr_samples_bg) == (1e-3, 512, 64, 1e-4, 32)
    assert hp.use_occupancy_grid and hp.use_color_calibration
    assert (hp.foreground_nr_iters_for_c2f, hp.background_nr_iters_for_c2f, hp.iter_finish_training) == (1, 10000, 200000)
    assert (OCC_NR_POINTS, OCC_DECAY, OCC_THRESH, OCC_EVERY, MASK_WEIGHT) == (256 * 256, 0.7, 1e-3, 8, 0.1)


@pytest.mark.parametrize("L", [6, 30, 32, 0])
def test_unsupported_level_counts_are_refused(L):
    from permuto_sdf_b200.nerf_train import NerfTrainer
    with pytest.raises(RuntimeError, match="nr_levels"):
        NerfTrainer(4, False, nr_levels=L)


def test_unknown_optimizer_is_refused():
    from permuto_sdf_b200.nerf_train import NerfTrainer
    with pytest.raises(RuntimeError, match="optimizer"):
        NerfTrainer(4, False, optimizer="sgd")


def _bare(with_mask, R_max=512):
    """a NerfTrainer shell with the state its input checks read (no device needed)"""
    from permuto_sdf_b200.nerf_train import NerfHyperParams, NerfTrainer
    tr = NerfTrainer.__new__(NerfTrainer)
    tr.hp, tr.with_mask = NerfHyperParams(), with_mask
    return tr


def test_input_refusals():
    tr = _bare(True)
    with pytest.raises(RuntimeError, match="mask"):
        tr._check_rays(512, False)
    with pytest.raises(RuntimeError, match="32-bit"):
        _bare(False)._check_rays(2 ** 24, True)
    with pytest.raises(RuntimeError, match="at least one ray"):
        _bare(False)._check_rays(0, True)
    assert _bare(False)._check_rays(512, False) == 512


def test_nerf_loss_is_train_nerf_formula():
    from permuto_sdf_b200.nerf_train import nerf_loss
    g = torch.Generator().manual_seed(0)
    gt, pred = torch.rand(16, 3, generator=g), torch.rand(16, 3, generator=g)
    hit = torch.rand(16, 1, generator=g) > 0.3
    ws, m = torch.rand(16, 1, generator=g), (torch.rand(16, 1, generator=g) > 0.5).float()
    loss, lr, lm = nerf_loss(gt, pred, hit, ws, m)
    want_rgb = (((gt - pred) ** 2) * hit.float()).sum() / 48
    want_m = -(m * torch.log(ws.clamp(1e-3, 1 - 1e-3)) + (1 - m) * torch.log(1 - ws.clamp(1e-3, 1 - 1e-3))).mean()
    assert torch.allclose(lr, want_rgb) and torch.allclose(lm, want_m) and torch.allclose(loss, want_rgb + 0.1 * want_m)
    assert nerf_loss(gt, pred, hit)[2] is None


def _problem(L, n, seed):
    g = torch.Generator().manual_seed(seed)
    T = 997
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [(2 * L + 4, 64), (64, 64), (64, 64), (64, 65), (80, 64), (64, 64), (64, 3)]
    W = [torch.randn(o, i, generator=g) / i ** 0.5 for i, o in dims]
    b = [torch.randn(o, generator=g) * 0.1 for _, o in dims]
    pos = torch.rand(n, 3, generator=g) - 0.5
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    return pos, dirs, lat, R.level_scales(L, 3), shift, R.window_of(L, 0.6), W, b, g


@pytest.mark.parametrize("L", [4, 24])
def test_oracle_at_d3_matches_fp64_autograd(L):
    """bg_reference / bg_forward_reference take the width from pos: at D = 3 the encoder gives 2L + 4 columns (concat {x, 0}), the
    gradients equal fp64 autograd and the forward values those of bg_reference, with finite positive error scales"""
    pos, dirs, lat, scale, shift, w, W, b, g = _problem(L, 50, L)
    g_rgb, g_den = torch.randn(50, 3, generator=g), torch.randn(50, 1, generator=g)
    ref = R.bg_reference(pos, dirs, lat, scale, shift, w, 1.0, W, b, g_rgb, g_den)
    glat, gW, gb = R.bg_autograd(pos, dirs, lat, scale, shift, w, 1.0, W, b, g_rgb, g_den)
    dense = R.dense_lattice(ref["lattice"])
    assert float((dense - glat).abs().max()) <= 1e-12 * max(1.0, float(glat.abs().max()))
    for l in range(7):
        assert float((ref["W"][l] - gW[l]).abs().max()) <= 1e-12 * max(1.0, float(gW[l].abs().max()))
        assert float((ref["b"][l] - gb[l]).abs().max()) <= 1e-12 * max(1.0, float(gb[l].abs().max()))
    fwd = R.bg_forward_reference(pos, dirs, lat, scale, shift, w, 1.0, W, b)
    assert torch.allclose(fwd["rgb_raw"], ref["rgb"].double(), rtol=0, atol=1e-12)
    assert torch.allclose(fwd["density"].reshape(-1), ref["density"].double().reshape(-1), rtol=0, atol=1e-12)
    for k in ("A_rgb", "A_density"):
        assert bool(torch.isfinite(fwd[k]).all()) and bool((fwd[k] > 0).all())


def test_oracle_error_scale_at_d3_bounds_a_perturbed_network():
    """A propagated at D = 3 covers the effect of rounding every weight to fp32-relative 2^-20: |delta out| <= 2^-20 A x a margin"""
    pos, dirs, lat, scale, shift, w, W, b, g = _problem(8, 64, 5)
    ref = R.bg_forward_reference(pos, dirs, lat, scale, shift, w, 1.0, W, b)
    eps = 2.0 ** -20
    Wp = [x * (1 + eps * (2 * torch.rand(x.shape, generator=g) - 1)) for x in W]
    bp = [x * (1 + eps * (2 * torch.rand(x.shape, generator=g) - 1)) for x in b]
    per = R.bg_forward_reference(pos, dirs, lat, scale, shift, w, 1.0, Wp, bp)
    for k, a in (("rgb_raw", "A_rgb"), ("density", "A_density")):
        ratio = float(((per[k] - ref[k]).abs() / (eps * ref[a])).max())
        assert ratio <= 4.0, (k, ratio)


REF_PY = os.path.join(os.environ.get("PERMUTO_SDF_REFERENCE") or "/root/reference", "permuto_sdf_py")


@pytest.mark.skipif(not os.path.isdir(REF_PY), reason="needs a checkout of the original project (PERMUTO_SDF_REFERENCE)")
def test_fixture_generator_reproduces_its_file(tmp_path):
    out = tmp_path / "nerf.npz"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, NERF_GOLDEN_OUT=str(out))
    subprocess.run([sys.executable, os.path.join(root, "tests", "golden", "make_nerf_golden.py")], check=True, env=env, cwd=root,
                   capture_output=True)
    a, b = np.load(os.path.join(root, "tests", "golden", "refpy_golden_nerf.npz")), np.load(out)
    assert sorted(a.keys()) == sorted(b.keys())
    for k in a.keys():
        assert np.array_equal(a[k], b[k]), k


def test_fixture_is_complete_and_small():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    path = os.path.join(root, "tests", "golden", "refpy_golden_nerf.npz")
    assert os.path.getsize(path) < 1 << 20
    G = np.load(path)
    for tag in ("nomask.", "mask."):
        for k in ("rgb", "density", "pred_rgb", "weights_sum", "bg_T", "loss", "grad.fg.encoding.lattice_values.rows", "grad.cal.bias"):
            assert tag + k in G, tag + k
    assert "nomask.grad.bg.mlp_rgb.4.weight" in G
