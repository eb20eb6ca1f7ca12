"""CPU checks of the image metrics (permuto_sdf_b200/metrics.py, csrc/image_metrics.cu): the numpy / fp64 oracle against an independent
torch-float64 statement of piq's psnr and ssim (F.avg_pool2d, the 2-D Gaussian through a grouped F.conv2d, then the formulas), cases with
a known answer, piq's pooling factor with its ties, the 8-bit quantization's ties to even, and the argument checks that need no device."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import image_metrics as om
from permuto_sdf_b200 import metrics


def piq_psnr(x, y):
    """piq.psnr(x, y, data_range=1.) in fp64"""
    return -10 * torch.log10(torch.mean((x - y) ** 2, dim=[1, 2, 3]) + 1e-8)


def piq_ssim(x, y, kernel_size=11, kernel_sigma=1.5, k1=0.01, k2=0.03):
    """piq.ssim(x, y, data_range=1.) in fp64: downsampling, gaussian_filter and _ssim_per_channel"""
    f = max(1, round(min(x.size()[-2:]) / 256))
    if f > 1:
        x, y = F.avg_pool2d(x, kernel_size=f), F.avg_pool2d(y, kernel_size=f)
    coords = torch.arange(kernel_size, dtype=x.dtype) - (kernel_size - 1) / 2.
    g = coords ** 2
    g = (-(g.unsqueeze(0) + g.unsqueeze(1)) / (2 * kernel_sigma ** 2)).exp()
    g /= g.sum()
    kernel = g.unsqueeze(0).repeat(x.size(1), 1, 1, 1)
    c1, c2, n = k1 ** 2, k2 ** 2, x.size(1)
    conv = lambda a: F.conv2d(a, weight=kernel, stride=1, padding=0, groups=n)
    mu_x, mu_y = conv(x), conv(y)
    mu_xx, mu_yy, mu_xy = mu_x ** 2, mu_y ** 2, mu_x * mu_y
    sigma_xx, sigma_yy, sigma_xy = conv(x ** 2) - mu_xx, conv(y ** 2) - mu_yy, conv(x * y) - mu_xy
    cs = (2. * sigma_xy + c2) / (sigma_xx + sigma_yy + c2)
    ss = (2. * mu_xy + c1) / (mu_xx + mu_yy + c1) * cs
    return ss.mean(dim=(-1, -2)).mean(1)


def images(B, C, H, W, seed, mask=False):
    rng = np.random.RandomState(seed)
    x = rng.rand(B, C, H, W).astype(np.float32)
    y = np.clip(x + 0.1 * rng.randn(B, C, H, W), 0, 1).astype(np.float32)
    m = (rng.rand(B, H, W) > 0.3).astype(np.float32) if mask else None
    return x, y, m


@pytest.mark.parametrize("B,C,H,W,f", [(2, 3, 37, 53, 1), (1, 1, 129, 67, 1), (2, 1, 385, 421, 2), (1, 3, 577, 769, 2),
                                       (1, 3, 1200, 1601, 5), (1, 1, 2049, 2051, 8)])
@pytest.mark.parametrize("mask,quantize_x", [(False, False), (True, True)])
def test_oracle_matches_piq_statement(B, C, H, W, f, mask, quantize_x):
    assert om.pool_factor(H, W) == f
    x, y, m = images(B, C, H, W, H + W, mask)
    xp, yp = om.prepare(x, y, m, quantize_x)
    tx, ty = torch.from_numpy(xp), torch.from_numpy(yp)
    np.testing.assert_allclose(om.psnr(x, y, m, quantize_x), piq_psnr(tx, ty).numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(om.ssim(x, y, m, quantize_x), piq_ssim(tx, ty).numpy(), rtol=0, atol=1e-12)


def test_identical_images_and_uniform_offset():
    x, _, _ = images(2, 3, 40, 50, 0)
    assert np.all(om.psnr(x, x) == 80.0)
    np.testing.assert_allclose(om.ssim(x, x), 1.0, rtol=0, atol=1e-14)
    # x a multiple of 2^-12 in [0, 0.5]: x + d is exact in fp32, so every difference is exactly d
    xq = (np.floor(x * 2048) / 4096).astype(np.float32)
    for d in (0.25, 0.015625, 2.0 ** -12):
        y = (xq + np.float32(d)).astype(np.float32)
        assert np.all(y - xq == np.float32(d))
        np.testing.assert_allclose(om.psnr(y, xq), -10 * np.log10(d * d + 1e-8), rtol=0, atol=1e-12)


@pytest.mark.parametrize("side,f", [(11, 1), (128, 1), (383, 1), (384, 2), (385, 2), (639, 2), (640, 2), (641, 3), (895, 3), (896, 4),
                                    (1152, 4), (1200, 5), (2048, 8)])
def test_pool_factor_rounds_half_to_even(side, f):
    assert om.pool_factor(side, side + 500) == f
    assert om.pool_factor(side + 7, side) == f
    assert metrics.pool_factor(side, 4 * side) == f


def _ties():
    """fp32 x in (0, 1) with fl32(x * 255) = k + 1/2 exactly, for as many k as exist"""
    out = []
    for k in range(255):
        c = np.float32((k + 0.5) / 255)
        for x in (np.nextafter(c, np.float32(0)), c, np.nextafter(c, np.float32(1))):
            if np.float32(x) * np.float32(255) == np.float32(k + 0.5):
                out.append((np.float32(x), k))
                break
    return out


def test_quantize_rounds_ties_to_even():
    ties = _ties()
    assert len(ties) > 100
    x = np.array([t for t, _ in ties], np.float32)
    k = np.array([k for _, k in ties])
    q = om.quantize(x)
    expect = np.where(k % 2 == 0, k, k + 1).astype(np.float32) / np.float32(255)
    assert np.array_equal(q, expect.astype(np.float32))
    # saturation at both ends, and exact levels stay
    assert np.array_equal(om.quantize(np.array([-0.3, 0.0, 1.0, 1.7, 128 / 255], np.float32)),
                          np.array([0, 0, 1, 1, np.float32(128) / np.float32(255)], np.float32))


def test_small_image_raises():
    x, y, _ = images(1, 3, 10, 40, 1)
    with pytest.raises(RuntimeError, match="smaller than"):
        om.ssim(x, y)
    x, y, _ = images(1, 1, 640, 21, 1)          # f = 1 (min 21), fine
    om.ssim(x, y)
    with pytest.raises(RuntimeError, match="smaller than"):
        metrics._check_ssim_size("ssim", 10, 400)
    metrics._check_ssim_size("ssim", 11, 11)


def test_metrics_refuse_host_tensors():
    x = torch.rand(1, 3, 20, 20)
    for fn in (metrics.psnr, metrics.ssim):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(x, x)
        with pytest.raises(RuntimeError, match="float32"):
            fn(x.double(), x.double())
        with pytest.raises(RuntimeError, match="B,C,H,W"):
            fn(x[0], x[0])


def test_workspace_bytes():
    lib = metrics.load_library()
    assert lib.psdf_image_metrics_workspace_bytes(0, 3, 10, 10) == -1
    assert lib.psdf_image_metrics_workspace_bytes(1, 3, -1, 10) == -1
    assert lib.psdf_image_metrics_workspace_bytes(65536, 3, 10, 10) == -3
    # 8 B per partial, the larger of the PSNR partials (ceil(H W / 2048), at most 1024) and the SSIM tiles of 8 x 32 positions:
    # 1200 x 1600 (f = 5): 938 and 29 x 10; 384 x 512 (f = 2): 96 and 23 x 8
    assert lib.psdf_image_metrics_workspace_bytes(16, 3, 1200, 1600) == 8 * 16 * 938
    assert lib.psdf_image_metrics_workspace_bytes(1, 1, 11, 11) == 8 * 1
    assert lib.psdf_image_metrics_workspace_bytes(2, 1, 384, 512) == 8 * 2 * 184
