"""numpy / fp64 restatement of the image metrics of evaluate_psnr.py (piq.psnr and piq.ssim at data_range = 1), as
include/psdf_b200.h states them for csrc/image_metrics.cu. Test infrastructure only.

Inputs: x, y [B,C,H,W] float32 (x the prediction), mask [B,H,W] or None. quantize_x: x = min(255, max(0, rne(x * 255))) / 255 in fp32
first (create_my_images.py's 8-bit PNG round trip); then x m and y m; everything after is fp64. The SSIM window is the 2-D Gaussian summed
directly (no separable passes)."""
import numpy as np

KERNEL_SIZE, SIGMA, K1, K2, EPS = 11, 1.5, 0.01, 0.03, 1e-8


def quantize(x):
    x = np.asarray(x, np.float32)
    k = np.minimum(np.float32(255), np.maximum(np.float32(0), np.rint(x * np.float32(255))))   # np.rint: ties to even
    return (k / np.float32(255)).astype(np.float32)


def prepare(x, y, mask=None, quantize_x=False):
    """-> (x, y) in fp64 after the optional quantization of x and the mask"""
    x = np.asarray(x, np.float32)
    y = np.asarray(y, np.float32)
    if quantize_x:
        x = quantize(x)
    x, y = x.astype(np.float64), y.astype(np.float64)
    if mask is not None:
        m = np.asarray(mask, np.float32).astype(np.float64)[:, None]
        x, y = x * m, y * m
    return x, y


def pool_factor(H, W):
    """piq: max(1, round(min(H, W) / 256)); Python's round is half to even"""
    return max(1, round(min(H, W) / 256))


def avg_pool(a, f):
    """F.avg_pool2d(a, f): f x f blocks with stride f, remainder dropped"""
    B, C, H, W = a.shape
    Hp, Wp = H // f, W // f
    return a[:, :, :Hp * f, :Wp * f].reshape(B, C, Hp, f, Wp, f).mean(axis=(3, 5))


def window():
    c = np.arange(KERNEL_SIZE, dtype=np.float64) - (KERNEL_SIZE - 1) / 2.0
    g = np.exp(-(c[None, :] ** 2 + c[:, None] ** 2) / (2 * SIGMA ** 2))
    return g / g.sum()


def filter_valid(a, g):
    """valid-mode window sums of a [B,C,H,W] with the 2-D window g, one term per tap"""
    k = g.shape[0]
    B, C, H, W = a.shape
    out = np.zeros((B, C, H - k + 1, W - k + 1))
    for i in range(k):
        for j in range(k):
            out += g[i, j] * a[:, :, i:i + H - k + 1, j:j + W - k + 1]
    return out


def psnr(x, y, mask=None, quantize_x=False):
    """-> [B] fp64"""
    x, y = prepare(x, y, mask, quantize_x)
    mse = ((x - y) ** 2).mean(axis=(1, 2, 3))
    return -10.0 * np.log10(mse + EPS)


def ssim(x, y, mask=None, quantize_x=False):
    """-> [B] fp64; raises RuntimeError when an image is smaller than the window after pooling"""
    x, y = prepare(x, y, mask, quantize_x)
    f = pool_factor(x.shape[2], x.shape[3])
    if f > 1:
        x, y = avg_pool(x, f), avg_pool(y, f)
    if x.shape[2] < KERNEL_SIZE or x.shape[3] < KERNEL_SIZE:
        raise RuntimeError("ssim: %d x %d after pooling by %d is smaller than the %d x %d window" % (x.shape[2], x.shape[3], f, KERNEL_SIZE,
                                                                                                    KERNEL_SIZE))
    g = window()
    c1, c2 = K1 ** 2, K2 ** 2
    mu_x, mu_y = filter_valid(x, g), filter_valid(y, g)
    mu_xx, mu_yy, mu_xy = mu_x ** 2, mu_y ** 2, mu_x * mu_y
    s_xx = filter_valid(x * x, g) - mu_xx
    s_yy = filter_valid(y * y, g) - mu_yy
    s_xy = filter_valid(x * y, g) - mu_xy
    cs = (2.0 * s_xy + c2) / (s_xx + s_yy + c2)
    ss = (2.0 * mu_xy + c1) / (mu_xx + mu_yy + c1) * cs
    return ss.mean(axis=(2, 3)).mean(axis=1)
