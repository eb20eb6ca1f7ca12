"""Image metrics on the GPU (csrc/image_metrics.cu): the PSNR and SSIM with which the reference's evaluate_psnr.py scores rendered frames
(piq.psnr and piq.ssim at data_range = 1), and the frame evaluation of `Trainer.evaluate` / `NerfTrainer.evaluate`.

    psnr(x, y, mask=None, quantize_x=False)     -> [B] fp64, -10 log10(mean (x - y)^2 + 1e-8)
    ssim(x, y, mask=None, quantize_x=False)     -> [B] fp64, piq's SSIM (11 x 11 Gaussian, sigma 1.5, average-pool downsampling)

x (the prediction) and y (the ground truth) are float32 [B,C,H,W] CUDA tensors, contiguous in NCHW or in channels-last order; mask [B,H,W]
multiplies both, as evaluate_psnr.py does (masked-out pixels count as exact matches). quantize_x first rounds x to 8 bits as the PNGs of
create_my_images.py are: min(255, max(0, rne(x * 255))) / 255 in fp32. That EasyPBR's to_cv8u is exactly this conversion (OpenCV's
convertTo(CV_8U, 255), which rounds half to even and saturates) is an assumption: its source is not available here, so it is unverified.
Everything after the quantization is fp64, and a call gives the same bits on every run. Nothing waits for the device."""
import torch

from ._lib import call, load_library

KERNEL_SIZE = 11
MAX_BATCH = 65535
_INT32_MAX = 2 ** 31 - 1
FRAME_ITER = 9999999              # create_my_images.py: iter_nr_for_anneal; cos_anneal_ratio = 1, forced_variance_finish


def pool_factor(H, W):
    """piq's downsampling factor max(1, round(min(H, W) / 256)), Python's round (half to even)"""
    return max(1, round(min(int(H), int(W)) / 256))


def _check_ssim_size(fn, H, W):
    f = pool_factor(H, W)
    if H // f < KERNEL_SIZE or W // f < KERNEL_SIZE:
        raise RuntimeError("%s: a %d x %d image is %d x %d after average pooling by %d, smaller than the %d x %d window"
                           % (fn, H, W, H // f, W // f, f, KERNEL_SIZE, KERNEL_SIZE))


def _layout(fn, name, t):
    """-> (tensor the kernel reads, nhwc flag): NCHW as it is, channels-last as its contiguous [B,H,W,C] permutation"""
    if t.is_contiguous():
        return t, 0
    if t.is_contiguous(memory_format=torch.channels_last):
        return t.permute(0, 2, 3, 1), 1
    raise RuntimeError("%s: %s must be contiguous in NCHW or channels-last order" % (fn, name))


def _run(entry, B, C, H, W, x, y, mask, quantize_x, out, ws):
    """entry(B, C, H, W, x, x_nhwc, y, y_nhwc, mask, quantize_x, out, workspace); x, y: (tensor, nhwc)"""
    call(entry, B, C, H, W, x[0], x[1], y[0], y[1], mask, 1 if quantize_x else 0, out, ws)


def _workspace(B, C, H, W, device):
    return torch.empty(int(load_library().psdf_image_metrics_workspace_bytes(B, C, H, W)), dtype=torch.uint8, device=device)


def _metric(fn, entry, x, y, mask, quantize_x):
    for name, t in (("x", x), ("y", y)):
        if not isinstance(t, torch.Tensor) or t.dim() != 4:
            raise RuntimeError("%s: %s must be a [B,C,H,W] tensor" % (fn, name))
        if t.dtype != torch.float32:
            raise RuntimeError("%s: %s must be float32, got %s" % (fn, name, t.dtype))
        if not t.is_cuda:
            raise RuntimeError("%s: %s must be on a CUDA device (there is no CPU path)" % (fn, name))
    if x.shape != y.shape:
        raise RuntimeError("%s: x and y must have the same shape, got %s and %s" % (fn, tuple(x.shape), tuple(y.shape)))
    if x.device != y.device:
        raise RuntimeError("%s: x and y must be on the same device, got %s and %s" % (fn, x.device, y.device))
    B, C, H, W = x.shape
    if min(B, C, H, W) < 1 or B > MAX_BATCH or max(C, H, W) > _INT32_MAX:
        raise RuntimeError("%s: shape %s not supported (every size at least 1, B at most %d)" % (fn, tuple(x.shape), MAX_BATCH))
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or tuple(mask.shape) != (B, H, W) or mask.dtype != torch.float32:
            raise RuntimeError("%s: mask must be a float32 [B,H,W] = [%d,%d,%d] tensor" % (fn, B, H, W))
        if mask.device != x.device:
            raise RuntimeError("%s: mask must be on the images' device %s, got %s" % (fn, x.device, mask.device))
        mask = mask.contiguous()
    if entry == "psdf_image_ssim":
        _check_ssim_size(fn, H, W)
    xs, ys = _layout(fn, "x", x), _layout(fn, "y", y)
    with torch.cuda.device(x.device):
        out = torch.empty(B, dtype=torch.float64, device=x.device)
        _run(entry, B, C, H, W, xs, ys, mask, quantize_x, out, _workspace(B, C, H, W, x.device))
    return out


def psnr(x, y, mask=None, quantize_x=False):
    """per-image PSNR in dB (piq.psnr, data_range = 1) of x against y after the optional quantization of x and the mask -> [B] fp64 on
    the device; an exact match gives 80 dB"""
    return _metric("psnr", "psdf_image_psnr", x, y, mask, quantize_x)


def ssim(x, y, mask=None, quantize_x=False):
    """per-image SSIM (piq.ssim, data_range = 1, kernel 11, sigma 1.5, k1 0.01, k2 0.03, average pooling by
    max(1, round(min(H, W) / 256))) of x against y after the optional quantization of x and the mask -> [B] fp64 on the device; raises
    when the pooled image is smaller than the window"""
    return _metric("ssim", "psdf_image_ssim", x, y, mask, quantize_x)


# ---------------------------------------------------------------------------------------------------- frames of a reel
def _reel(fn, tensor_reel):
    rgb = tensor_reel.rgb_reel
    if rgb.dim() != 4 or rgb.shape[1] != 3:
        raise RuntimeError("%s: the reel's rgb must be [I,3,H,W], got %s" % (fn, tuple(rgb.shape)))
    I, _, H, W = rgb.shape
    if H * W > _INT32_MAX:
        raise RuntimeError("%s: a %d x %d frame has more pixels than the ray kernel indexes in 32 bits" % (fn, H, W))
    return I, H, W


def _image_indices(fn, image_indices, I):
    idx = [int(i) for i in image_indices]
    bad = [i for i in idx if not 0 <= i < I]
    if bad:
        raise RuntimeError("%s: image index %d outside the reel's %d images" % (fn, bad[0], I))
    return idx


def render_frame(fn, tensor_reel, img_idx, models, render):
    """every pixel of image img_idx of a TensorReel as one ray (PermutoSDF.rays_from_reel_indices with pix = arange(H W)), rendered by
    render(ray_origins, ray_dirs) with every module of `models` in eval mode. The modules' train flags and the models' last_iter_nr
    (which the coarse-to-fine windows record) are restored afterwards. -> (render's result, H, W)"""
    from .permuto_sdf import PermutoSDF
    I, H, W = _reel(fn, tensor_reel)
    i = _image_indices(fn, [img_idx], I)[0]
    dev = tensor_reel.rgb_reel.device
    pix = torch.arange(H * W, dtype=torch.int32, device=dev)
    img = torch.full((H * W,), i, dtype=torch.int32, device=dev)
    o, d, _, _, _ = PermutoSDF.rays_from_reel_indices(tensor_reel, pix, img)
    models = [m for m in models if m is not None]
    flags = [(m, m.training) for model in models for m in model.modules()]
    iters = [(m, m.last_iter_nr) for m in models if hasattr(m, "last_iter_nr")]
    try:
        for m, _ in flags:
            m.training = False
        out = render(o, d)
    finally:
        for m, t in flags:
            m.training = t
        for m, it in iters:
            m.last_iter_nr = it
    return out, H, W


def image(rows, H, W):
    """[H W, C] rows of a frame -> the reference's [1,C,H,W] image (a channels-last view of the rows)"""
    return rows.view(H, W, -1).permute(2, 0, 1).unsqueeze(0)


def evaluate_frames(fn, tensor_reel, image_indices, quantize, models, render_rgb):
    """create_my_images.py + evaluate_psnr.py for the images `image_indices` (None: all) of a TensorReel: each frame's rgb rows from
    render_frame(fn, tensor_reel, i, models, render_rgb) (render_rgb(o, d) -> [H W, 3]), 8-bit quantized when `quantize`, scored with psnr and
    ssim against the reel's rgb, both multiplied by the reel's mask when it has one. The rows go to the kernels as NHWC and the reel as NCHW,
    with no copies. The ray kernel's ground truth is not used: it is already multiplied by the mask, and evaluate_psnr.py multiplies once.
    -> {"image_indices", "psnr", "ssim" (fp64 per image, on the host), "psnr_mean", "ssim_mean"}; the means are of the per-image values, as
    evaluate_psnr.py's EvalResultsPerScene takes them. One host sync, at the end."""
    I, H, W = _reel(fn, tensor_reel)
    _check_ssim_size(fn, H, W)
    idx = list(range(I)) if image_indices is None else _image_indices(fn, image_indices, I)
    if not idx:
        raise RuntimeError("%s: no image to evaluate" % fn)
    rgb = tensor_reel.rgb_reel
    if rgb.dtype != torch.float32 or not rgb.is_contiguous():
        raise RuntimeError("%s: the reel's rgb must be a contiguous float32 tensor" % fn)
    mask = getattr(tensor_reel, "mask_reel", None)
    mask = mask if mask is not None and mask.numel() > 0 else None
    if mask is not None and (mask.dtype != torch.float32 or not mask.is_contiguous() or tuple(mask.shape) != (I, 1, H, W)):
        raise RuntimeError("%s: the reel's mask must be a contiguous float32 [I,1,H,W] tensor" % fn)
    dev = rgb.device
    with torch.cuda.device(dev):
        ps = torch.empty(len(idx), dtype=torch.float64, device=dev)
        ss = torch.empty(len(idx), dtype=torch.float64, device=dev)
        ws = _workspace(1, 3, H, W, dev)
        for k, i in enumerate(idx):
            rows, _, _ = render_frame(fn, tensor_reel, i, models, render_rgb)
            args = (1, 3, H, W, (rows.contiguous(), 1), (rgb[i:i + 1], 0), None if mask is None else mask[i], quantize)
            _run("psdf_image_psnr", *args, ps[k:k + 1], ws)
            _run("psdf_image_ssim", *args, ss[k:k + 1], ws)
        ps, ss = ps.cpu(), ss.cpu()
    p, s = ps.tolist(), ss.tolist()
    return {"image_indices": idx, "psnr": ps, "ssim": ss, "psnr_mean": sum(p) / len(p), "ssim_mean": sum(s) / len(s)}
