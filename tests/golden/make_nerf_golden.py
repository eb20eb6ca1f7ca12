"""Fixture generator for the NeRF training iteration: runs the reference's UNMODIFIED NerfHash (permuto_sdf_py/models/models.py) as the
foreground NerfHash(3) and the background NerfHash(4), Colorcal, VolumeRenderingNerf (volume_rendering/volume_rendering_modules.py) and
the losses of train_nerf.py on the CPU through oracle/refpy.py, and stores seeded inputs, parameters, outputs, the loss and every parameter
gradient, without and with mask, in tests/golden/refpy_golden_nerf.npz. Needs a checkout of the original project, named by
PERMUTO_SDF_REFERENCE; tests/test_nerf_train_gpu.py loads the .npz and compares the CUDA paths.

    python tests/golden/make_nerf_golden.py

The hash tables are regenerated from seeds on both sides (make_refpy_golden.lattice_from_seed); table gradients are stored sparsely.
The gradients are those of the reference's kernels as they are, including integrate_with_weights_backward's read of the green channel
for the blue one in the weight gradient (SURVEY.md A.12); the tests compare them in the same mode.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_refpy_golden import lattice_from_seed, sparse_rows, unit  # noqa: E402

L, T, F = 24, 2 ** 18, 2
SEED_FG, SEED_BG = 21, 23
ITER = 5000                      # background window mid-ramp (background_nr_iters_for_c2f 10000), foreground window open
R, NIMG, NB = 32, 4, 6


def inputs():
    """seeded rays, packed foreground samples (ragged, with empty rays) and NB background samples per ray"""
    g = torch.Generator().manual_seed(77)
    cam = unit(torch.randn(R, 3, generator=g)) * 1.2
    tgt = torch.randn(R, 3, generator=g) * 0.25
    tgt[:4] = cam[:4] * 2.0                                  # rays that point away: no hit
    dirs = unit(tgt - cam)
    cnt = torch.randint(0, 11, (R,), generator=g)
    cnt[:6:2] = 0
    end = torch.cumsum(cnt, 0)
    se = torch.stack([end - cnt, end], 1).to(torch.int32)
    N = int(end[-1])
    ray_of = torch.repeat_interleave(torch.arange(R), cnt)
    fg_pos = (torch.rand(N, 3, generator=g) - 0.5) * 0.8
    fg_dirs = dirs[ray_of].clone()
    fg_dt = torch.rand(N, 1, generator=g) * 0.03 + 1e-3
    Nb = NB * R
    bg_pos4 = torch.cat([unit(torch.randn(Nb, 3, generator=g)), torch.rand(Nb, 1, generator=g)], 1)
    bg_dirs = dirs.repeat_interleave(NB, 0).clone()
    bg_dt = torch.rand(Nb, 1, generator=g) * 0.2 + 1e-3
    bg_se = torch.stack([torch.arange(R) * NB, torch.arange(R) * NB + NB], 1).to(torch.int32)
    gt = torch.rand(R, 3, generator=g)
    mask = (torch.rand(R, 1, generator=g) > 0.4).float()
    img = torch.randint(0, NIMG, (R,), generator=g).to(torch.int32)
    return dict(origins=cam, dirs=dirs, fg_se=se, fg_pos=fg_pos, fg_dirs=fg_dirs, fg_dt=fg_dt, bg_se=bg_se, bg_pos4=bg_pos4, bg_dirs=bg_dirs,
                bg_dt=bg_dt, gt=gt, mask=mask, img=img)


def main():
    from oracle import refpy
    M = refpy.install()
    import permuto_sdf as ps                    # the CPU stand-ins installed above
    torch.manual_seed(4321)
    aabb = ps.Sphere(0.5, [0, 0, 0])
    fg_m = M.NerfHash(3, boundary_primitive=aabb, nr_iters_for_c2f=1)
    bg_m = M.NerfHash(4, boundary_primitive=aabb, nr_iters_for_c2f=10000)
    cal = M.Colorcal(NIMG, 0)
    with torch.no_grad():
        fg_m.encoding.lattice_values.copy_(lattice_from_seed(SEED_FG, L, T, F, 0.3))
        bg_m.encoding.lattice_values.copy_(lattice_from_seed(SEED_BG, L, T, F, 0.3))
        fg_m.mlp_feat_and_density[-1].bias.add_(torch.randn(65) * 0.5)     # a spread of densities
        cal.weight_delta.normal_(0, 0.1)
        cal.bias.normal_(0, 0.1)
    out = {}
    for prefix, m in (("fg.", fg_m), ("bg.", bg_m), ("cal.", cal)):
        for k, v in m.state_dict().items():
            if "lattice_values" not in k:
                out[prefix + k] = v.detach().numpy().copy()
    I = inputs()
    out.update({"in." + k: v.numpy() for k, v in I.items()})
    _, _, _, _, hit = aabb.ray_intersection(I["origins"], I["dirs"])

    def packed(se, pos, dirs, dt, four_d):
        n = pos.shape[0]
        rsp = ps.RaySamplesPacked(se.shape[0], n)
        rsp.ray_start_end_idx = se.clone()
        if four_d:
            rsp.samples_pos_4d = pos.clone()
        else:
            rsp.samples_pos = pos.clone()
        rsp.samples_dirs, rsp.samples_dt = dirs.clone(), dt.clone()
        return rsp

    fg = packed(I["fg_se"], I["fg_pos"], I["fg_dirs"], I["fg_dt"], False)
    bg = packed(I["bg_se"], I["bg_pos4"], I["bg_dirs"], I["bg_dt"], True)
    for tag, with_mask in (("nomask", False), ("mask", True)):
        for m in (fg_m, bg_m, cal):
            m.zero_grad()
        # train_nerf.py:61-95 (run_net) and :176-182 (losses)
        rgb, density = fg_m(fg.samples_pos, fg.samples_dirs, ITER, cal, I["img"], ray_start_end_idx=fg.ray_start_end_idx)
        weights, weights_sum, bg_T = fg_m.volume_renderer_nerf.compute_weights(fg, density.view(-1, 1))
        pred_rgb = fg_m.volume_renderer_nerf.integrate(fg, rgb, weights)
        if not with_mask:
            rgb_bg, density_bg = bg_m(bg.samples_pos_4d, bg.samples_dirs, ITER, cal, I["img"], ray_start_end_idx=bg.ray_start_end_idx)
            weights_bg, _, _ = bg_m.volume_renderer_nerf.compute_weights(bg, density_bg.view(-1, 1))
            pred_rgb_bg = bg_m.volume_renderer_nerf.integrate(bg, rgb_bg, weights_bg)
            pred_rgb = pred_rgb + bg_T.view(-1, 1) * pred_rgb_bg
        loss = ((I["gt"] - pred_rgb) ** 2 * hit * 1.0).mean()
        if with_mask:
            loss = loss + torch.nn.functional.binary_cross_entropy(weights_sum.clip(1e-3, 1.0 - 1e-3), I["mask"]) * 0.1
        loss.backward()
        p = tag + "."
        out.update({p + "rgb": rgb.detach().numpy(), p + "density": density.detach().numpy(), p + "pred_rgb": pred_rgb.detach().numpy(),
                    p + "weights_sum": weights_sum.detach().numpy(), p + "bg_T": bg_T.detach().numpy(), p + "loss": loss.detach().numpy().reshape(1)})
        for mp, m in (("fg.", fg_m), ("bg.", bg_m), ("cal.", cal)):
            for k, prm in m.named_parameters():
                if prm.grad is None:
                    continue
                key = p + "grad." + mp + k
                if "lattice_values" in k:
                    out[key + ".rows"], out[key + ".vals"] = sparse_rows(prm.grad)
                else:
                    out[key] = prm.grad.numpy().copy()
    path = os.environ.get("NERF_GOLDEN_OUT") or os.path.join(ROOT, "tests", "golden", "refpy_golden_nerf.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
