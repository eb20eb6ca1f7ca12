"""Image metrics on the GPU (csrc/image_metrics.cu, permuto_sdf_b200/metrics.py) against the fp64 oracle (oracle/image_metrics.py) at
sizes from the 11 x 11 minimum to 2048 x 2048, in both layouts, with and without a mask and the 8-bit quantization; the same bits on every
call; argument errors raised before anything is launched. Then `render_frame` and `evaluate` of Trainer (with a mask, and without one on the
fused background) and NerfTrainer on synthetic reels: evaluate equals render_frame + quantization + the oracle, render_frame equals render
on the same rays, nothing of the trainer changes, and a reel whose rgb is the rendered frame scores exactly 80 dB and SSIM 1."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import scenes
from oracle import image_metrics as om
from test_volume_render_gpu import _same, _state, _trained

pytestmark = pytest.mark.gpu
TOL = 1e-10


def _images(B, C, H, W, seed):
    rng = np.random.RandomState(seed)
    x = rng.rand(B, C, H, W).astype(np.float32)
    y = np.clip(x + 0.05 * rng.randn(B, C, H, W), 0, 1).astype(np.float32)
    m = (rng.rand(B, H, W) > 0.3).astype(np.float32)
    return x, y, m


def _layouts(a):
    t = torch.from_numpy(a).cuda()
    return {"nchw": t, "nhwc": t.contiguous(memory_format=torch.channels_last)}


@pytest.mark.parametrize("H,W", [(11, 11), (17, 300), (384, 512), (1200, 1600), (2048, 2048)])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("C", [1, 3])
def test_kernels_match_oracle(cuda, H, W, B, C):
    from permuto_sdf_b200 import metrics
    x, y, m = _images(B, C, H, W, H * 7 + W + B + C)
    xs, ys, mt = _layouts(x), _layouts(y), torch.from_numpy(m).cuda()
    for mask in (None, m):
        for q in (False, True):
            want = {"psnr": om.psnr(x, y, mask, q), "ssim": om.ssim(x, y, mask, q)}
            for lx in xs:
                for ly in ys:
                    for name, fn in (("psnr", metrics.psnr), ("ssim", metrics.ssim)):
                        got = fn(xs[lx], ys[ly], None if mask is None else mt, q)
                        assert got.dtype == torch.float64 and got.shape == (B,)
                        err = np.abs(got.cpu().numpy() - want[name]).max()
                        assert err <= TOL, (name, lx, ly, mask is not None, q, err)


def test_same_bits_on_every_call(cuda):
    from permuto_sdf_b200 import metrics
    x, y, m = _images(3, 3, 1200, 1600, 5)
    x, y, m = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), torch.from_numpy(m).cuda()
    for fn in (metrics.psnr, metrics.ssim):
        a, b = fn(x, y, m, True), fn(x, y, m, True)
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_known_answers(cuda):
    from permuto_sdf_b200 import metrics
    x = torch.rand(2, 3, 64, 80, device="cuda")
    assert metrics.psnr(x, x).tolist() == [80.0, 80.0]
    assert metrics.ssim(x, x).tolist() == [1.0, 1.0]
    # fp32 values with x * 255 = k + 1/2 exactly round to the even neighbour
    from test_image_metrics_cpu import _ties
    ties = _ties()
    k = np.array([t[1] for t in ties])
    xt = torch.tensor([t[0] for t in ties], dtype=torch.float32, device="cuda").view(1, 1, 1, -1)
    want = torch.from_numpy((np.where(k % 2 == 0, k, k + 1).astype(np.float32) / np.float32(255)).astype(np.float32)).cuda().view(1, 1, 1, -1)
    assert metrics.psnr(xt, want, quantize_x=True).tolist() == [80.0]
    assert metrics.psnr(xt, want).tolist()[0] < 80.0


def test_argument_errors_before_any_launch(cuda):
    from permuto_sdf_b200 import _lib, metrics
    x = torch.rand(2, 3, 40, 50, device="cuda")
    m = torch.ones(2, 40, 50, device="cuda")
    bad = [((x, x[:1]), "same shape"), ((x, x.double()), "float32"), ((x, x.cpu()), "CUDA"), ((x[0], x[0]), "B,C,H,W"),
           ((x, x, m[:1]), "mask"), ((x, x, m.double()), "mask"), ((x, x, m.cpu()), "device"), ((x[:, :, ::2], x[:, :, ::2]), "contiguous")]
    if torch.cuda.device_count() > 1:
        bad.append(((x, x.to("cuda:1")), "same device"))
    _lib.stats_begin()
    try:
        for fn in (metrics.psnr, metrics.ssim):
            for args, msg in bad:
                with pytest.raises(RuntimeError, match=msg):
                    fn(*args)
        small = torch.rand(1, 3, 10, 400, device="cuda")
        with pytest.raises(RuntimeError, match="smaller than"):
            metrics.ssim(small, small)
    finally:
        calls, _, _ = _lib.stats_end()
    assert calls == {}
    metrics.psnr(small, small)                   # PSNR has no minimum size


# ------------------------------------------------------------------------------------------------ trainers
class _Reel:
    def __init__(self, nimg, H, W, with_mask, seed=3):
        rgb, mask, K, tf = scenes.synthetic_reel(nimg, H, W, seed)
        K[:, 0, 0] *= W / 80.0
        K[:, 1, 1] *= W / 80.0
        self.rgb_reel, self.K_reel, self.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, K, tf)]
        self.mask_reel = torch.from_numpy(mask).cuda() if with_mask else None


def _sdf_trainer(with_mask):
    tr = _trained(16, 64, with_mask)
    for m in (tr.model_sdf, tr.model_rgb, tr.model_bg):
        if m is not None:
            m.train()                  # render_frame and evaluate switch to eval mode and back
    return tr


def _nerf_trainer():
    from permuto_sdf_b200.nerf_train import NerfTrainer
    tr = NerfTrainer(2, False, nr_levels=16, capacity=2 ** 14)
    reel = _Reel(2, 60, 80, False)
    g = torch.Generator().manual_seed(0)
    for _ in range(3):
        pix = torch.randint(0, 60 * 80, (512,), generator=g).to(torch.int32).cuda()
        img = torch.randint(0, 2, (512,), generator=g).to(torch.int32).cuda()
        tr.step_from_reel(reel, pix, img)
    return tr


def _models(tr):
    return [m for m in (getattr(tr, "model_sdf", None), getattr(tr, "model_rgb", None), getattr(tr, "model", None), tr.model_bg,
                        tr.model_colorcal) if m is not None]


def _nerf_state(tr):
    from permuto_sdf import OccupancyGrid, RaySampler
    params = [p for m in _models(tr) for p in m.parameters()]
    g = tr.occupancy_grid
    return dict(params=[p.detach().clone() for p in params], grads=[None if p.grad is None else p.grad.clone() for p in params],
                grid=(g.get_grid_values().clone(), g.get_grid_occupancy().clone()), rng=[(r.state, r.inc) for r in (OccupancyGrid.m_rng,
                                                                                                                   RaySampler.m_rng)],
                torch_rng=(torch.get_rng_state(), torch.cuda.get_rng_state()), counters=tr.iter_nr)


def _full_state(tr):
    st = _state(tr) if hasattr(tr, "params") else _nerf_state(tr)
    st["flags"] = [[m.training for m in model.modules()] for model in _models(tr)]
    st["last_iter_nr"] = [getattr(m, "last_iter_nr", None) for m in _models(tr)]
    return st


def _render_eval(tr, o, d):
    """render() with the models in eval mode, as create_my_images.py renders -> (rgb, normals or None, weights sum)"""
    models = _models(tr)
    for m in models:
        m.eval()
    try:
        if hasattr(tr, "params"):
            rgb, _, n, w = tr.render(o, d, None, 9999999, 1.0, tr.hp.forced_variance_finish)
            return rgb, n, w
        rgb, _, w = tr.render(o, d)
        return rgb, None, w
    finally:
        for m in models:
            m.train()


CASES = [("sdf_mask", True), ("sdf_bg", False), ("nerf", True)]


@pytest.mark.parametrize("kind,reel_mask", CASES)
@pytest.mark.parametrize("H,W", [(60, 80), (400, 520)])
def test_render_frame_and_evaluate(cuda, kind, reel_mask, H, W):
    from permuto_sdf_b200.permuto_sdf import PermutoSDF
    tr = _nerf_trainer() if kind == "nerf" else _sdf_trainer(kind == "sdf_mask")
    reel = _Reel(2, H, W, reel_mask)
    before = _full_state(tr)
    res = tr.evaluate(reel)
    frames = [tr.render_frame(reel, i) for i in range(2)]
    torch.cuda.synchronize()
    assert _same(before, _full_state(tr))
    assert res["image_indices"] == [0, 1]
    assert res["psnr"].dtype == torch.float64 and res["psnr"].device.type == "cpu"
    for k, fr in enumerate(frames):
        rgb, wsum = fr[0], fr[-1]
        assert rgb.shape == (1, 3, H, W) and wsum.shape == (1, 1, H, W)
        # evaluate = render_frame, then the 8-bit round trip in torch, then the oracle
        # (a tensor divisor: torch divides by a scalar as a product with its reciprocal, which is not always the rounded quotient)
        k8 = torch.clamp(torch.round(rgb * 255), 0, 255)
        xq = (k8 / torch.full_like(k8, 255.0)).contiguous().cpu().numpy()
        y = reel.rgb_reel[k:k + 1].cpu().numpy()
        m = None if reel.mask_reel is None else reel.mask_reel[k].cpu().numpy()
        assert abs(float(res["psnr"][k]) - om.psnr(xq, y, m)[0]) <= TOL
        assert abs(float(res["ssim"][k]) - om.ssim(xq, y, m)[0]) <= TOL
        # render_frame = render in eval mode on the frame's rays
        pix = torch.arange(H * W, dtype=torch.int32, device="cuda")
        o, d, _, _, _ = PermutoSDF.rays_from_reel_indices(reel, pix, torch.full_like(pix, k))
        ref_rgb, ref_n, ref_w = _render_eval(tr, o, d)
        assert torch.equal(rgb.permute(0, 2, 3, 1).reshape(-1, 3), ref_rgb)
        assert torch.equal(wsum.permute(0, 2, 3, 1).reshape(-1, 1), ref_w)
        if ref_n is not None:
            R = torch.linalg.inv(reel.tf_world_cam_reel[k].cpu())[0:3, 0:3].cuda()
            want = F.normalize(torch.matmul(R, ref_n.t()).t(), dim=1)
            assert torch.equal(fr[1].permute(0, 2, 3, 1).reshape(-1, 3), want)
            assert float(want.norm(dim=1).max()) <= 1 + 1e-6
    assert res["psnr_mean"] == sum(res["psnr"].tolist()) / 2 and res["ssim_mean"] == sum(res["ssim"].tolist()) / 2
    # the rendered frame as ground truth: an exact match
    reel.rgb_reel = torch.cat([fr[0] for fr in frames]).contiguous()
    exact = tr.evaluate(reel, quantize=False)
    assert exact["psnr"].tolist() == [80.0, 80.0] and exact["ssim"].tolist() == [1.0, 1.0]
    one = tr.evaluate(reel, image_indices=[1], quantize=False)
    assert one["image_indices"] == [1] and one["psnr_mean"] == 80.0


def test_evaluate_refuses_before_rendering(cuda):
    from permuto_sdf_b200 import _lib
    tr = _sdf_trainer(True)
    reel = _Reel(2, 60, 80, True)
    _lib.stats_begin()
    try:
        with pytest.raises(RuntimeError, match="image index 2"):
            tr.evaluate(reel, image_indices=[0, 2])
        with pytest.raises(RuntimeError, match="image index -1"):
            tr.render_frame(reel, -1)
        small = _Reel(1, 10, 80, True)
        with pytest.raises(RuntimeError, match="smaller than"):
            tr.evaluate(small)
    finally:
        calls, _, _ = _lib.stats_end()
    assert calls == {}
