"""Volume-rendered frames on the fused kernels: `Trainer.render`, the counterpart of `run_net_in_chunks` (train_permuto_sdf.py:172-209),
which renders every PSNR, orbit and novel-view image of the reference (create_my_images.py:151, render_orbit.py, render_from_frame.py).

`run_net_in_chunks` evaluates the SDF through the per-op encoder under torch.autograd (get_sdf_and_gradient with create_graph) and
composites with per-op kernels. Here one chunk of rays is the sequence

    run_net_samples                     occupancy-grid samples + 2 importance rounds (the code of run_net; one host sync per compaction)
    psdf_sdf_fused_forward              sdf, d sdf/dx and geometric feature at the samples (value + tangent forward)                1
    psdf_rgb_fused_forward              raw colour (weights Lipschitz-normalised and packed once per render call)                 1
    psdf_bg_fused_forward               background NerfHash, scenes without masks only                                              1
    psdf_nerf_bg_composite_forward      background compositing (sigmoid folded in, no calibration)                                  1
    psdf_neus_render_forward            NeuS compositing: colour, normals, weights sum, background blend (colour head folded in)    1

The outputs are written straight into full-frame tensors. Sample counts differ from chunk to chunk (the reference's exact-size compaction);
the per-sample workspaces are kept between chunks and calls and grow only when a chunk needs more rows.

Size limit: the samplers, the compaction, importance resampling and the compositing kernels index per-sample rows with 32-bit ints (at
most 4 floats per row; the fused network kernels use 64-bit offsets). A chunk holds at most chunk * (max_nr_samples_per_ray +
2 nr_samples_imp_sampling) foreground samples at every stage of the sampling and chunk * nr_samples_bg background samples; render() keeps
both <= MAX_SAMPLES_PER_CHUNK = 2^26, so every such index stays below 4 * 2^26 = 2^28 < 2^31 and the warp-per-ray kernels' thread index
(32 * rays <= 2^31) below 2^32. With the default hyper-parameters (96 samples per ray) that is 699 050 rays per chunk."""
import math

import torch

from ._lib import call

MAX_SAMPLES_PER_CHUNK = 1 << 26
DEFAULT_CHUNK = 1 << 16


class VolumeRender:
    def __init__(self, trainer):
        self.tr = trainer
        self._ws = {}

    @staticmethod
    def unsupported_reason(tr):
        if getattr(tr.model_sdf, "fused", None) is None:
            return "the SDF model is not on the fused kernels (Trainer(fused_inference=True) puts it there)"
        if getattr(tr.model_rgb, "fused", None) is None:
            return "the colour model is not on the fused kernels (Trainer(fused_inference=True, fused_training=True) puts it there)"
        if tr.model_bg is not None and getattr(tr.model_bg, "fused", None) is None:
            return "background model (no --with_mask) on the per-op kernels (Trainer(fused_background=True) fuses it)"
        return None

    @staticmethod
    def max_chunk(hp):
        """largest chunk_size whose samples stay within MAX_SAMPLES_PER_CHUNK"""
        per_ray = int(hp.max_nr_samples_per_ray) + (2 * int(hp.nr_samples_imp_sampling) if hp.do_importance_sampling else 0)
        return MAX_SAMPLES_PER_CHUNK // max(per_ray, int(hp.nr_samples_bg), 1)

    def _buf(self, name, rows, cols, dev):
        """rows x cols view of a persistent workspace that grows (by at least a quarter) when a chunk needs more rows"""
        t = self._ws.get(name)
        if t is None or t.shape[0] < rows or t.device != dev:
            cap = max(rows, 1) if t is None else max(rows, t.shape[0] + t.shape[0] // 4)
            t = self._ws[name] = torch.empty(cap, cols, device=dev)
        return t[:rows]

    @torch.no_grad()
    def render(self, ray_origins, ray_dirs, chunk_size, iter_nr_for_anneal, cos_anneal_ratio, forced_variance):
        from .train import run_net_samples
        tr = self.tr
        hp = tr.hp
        why = self.unsupported_reason(tr)
        if why is not None:
            raise RuntimeError("Trainer.render: " + why)
        chunk_size = int(chunk_size)
        if not 1 <= chunk_size <= self.max_chunk(hp):
            raise ValueError("Trainer.render: chunk_size must be in [1, %d] (at most %d samples per chunk), got %d"
                             % (self.max_chunk(hp), MAX_SAMPLES_PER_CHUNK, chunk_size))
        R = ray_origins.shape[0]
        dev = ray_origins.device
        m_sdf, m_rgb, m_bg = tr.model_sdf, tr.model_rgb, tr.model_bg
        fs, fr = m_sdf.fused, m_rgb.fused
        pred_rgb = torch.empty(R, 3, device=dev)
        pred_rgb_bg = torch.empty(R, 3, device=dev) if m_bg is not None else None
        pred_normals = torch.empty(R, 3, device=dev)
        weights_sum = torch.empty(R, 1, device=dev)
        if R == 0:
            return pred_rgb, pred_rgb_bg, pred_normals, weights_sum
        it = iter_nr_for_anneal
        # ---- per call: weights -> operand blobs, coarse-to-fine windows, inv_s (SingleVarianceNetwork.forward without its state)
        if fs._versions != fs._cur_versions():
            fs.repack()
        enc, enc_c = m_sdf.encoding, m_rgb.encoding
        win = m_sdf.window(it).view(-1).contiguous()
        sdf_args = (enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(), win, enc.concat_points_scaling, fs.hidden, fs.out_dim,
                    fs.blob)
        L, c = fr.layers, m_rgb.mlp.lipshitz_bound_per_layer
        call("psdf_lipschitz_pack4", fr.in_dim, *fr.h, 3, L[0].weight.detach(), L[0].bias.detach(), c[0].detach(), L[1].weight.detach(),
             L[1].bias.detach(), c[1].detach(), L[2].weight.detach(), L[2].bias.detach(), c[2].detach(), L[3].weight.detach(),
             L[3].bias.detach(), c[3].detach(), fr.blob)
        win_c = fr._window(it)
        rgb_args = (enc_c.lattice_values.detach(), enc_c.scale_factor, enc_c.shift_tensor(), win_c, enc_c.concat_points_scaling, *fr.h, fr.blob)
        variance = m_rgb.volume_renderer_neus.deviation_network.variance
        if forced_variance is not None:
            inv_s = torch.exp(torch.ones((), device=variance.device) * forced_variance * 10.0)
        else:
            inv_s = torch.exp(variance.detach() * 10.0)
        inv_s = inv_s.reshape(1).float().contiguous()
        if m_bg is not None:
            fb, enc_b = m_bg.fused, m_bg.encoding
            fb.pack(fb.params())
            bg_args = (enc_b.lattice_values.detach(), enc_b.scale_factor, enc_b.shift_tensor(), fb._window(it), enc_b.concat_points_scaling,
                       fb.blob)
        # ---- per chunk (the split of run_net_in_chunks: ceil(R / chunk_size) chunks of equal size)
        nr_chunks = max(1, math.ceil(R / chunk_size))
        step = math.ceil(R / nr_chunks)
        for a in range(0, R, step):
            b = min(a + step, R)
            o, d = ray_origins[a:b].contiguous(), ray_dirs[a:b].contiguous()
            fg, bg = run_net_samples(hp.with_mask, hp, o, d, m_sdf, tr.occupancy_grid, it)
            N = fg.samples_pos.shape[0]
            sdf, grad = self._buf("sdf", N, 1, dev), self._buf("grad", N, 3, dev)
            geom, x_raw = self._buf("geom", N, fs.out_dim - 1, dev), self._buf("x_raw", N, 3, dev)
            if N > 0:
                call("psdf_sdf_fused_forward", N, enc.nr_levels, enc.capacity, fg.samples_pos, *sdf_args, sdf, grad, geom)
                call("psdf_rgb_fused_forward", N, enc_c.nr_levels, enc_c.capacity, fg.samples_pos, fg.samples_dirs, grad, geom, geom.shape[1],
                     *rgb_args, x_raw)
            bg_rgb = None
            if m_bg is not None and bg is not None and bg.samples_pos_4d.shape[0] != 0:
                Nb = bg.samples_pos_4d.shape[0]
                bx, bd, bg_rgb = self._buf("bg_x", Nb, 3, dev), self._buf("bg_density", Nb, 1, dev), self._buf("bg_rgb", b - a, 3, dev)
                call("psdf_bg_fused_forward", Nb, enc_b.nr_levels, enc_b.capacity, bg.samples_pos_4d, bg.samples_dirs, *bg_args, bx, bd)
                call("psdf_nerf_bg_composite_forward", *bg._rsp(), bx, bd.view(-1), bg.samples_dt.view(-1).contiguous(), None, None, None, -1,
                     bg_rgb)
            call("psdf_neus_render_forward", *fg._rsp(), sdf.view(-1), grad, x_raw, fg.samples_dirs, fg.samples_dt, inv_s, float(cos_anneal_ratio),
                 None, None, None, -1, bg_rgb, pred_rgb[a:b], pred_rgb_bg[a:b] if bg_rgb is not None else None, pred_normals[a:b],
                 weights_sum[a:b])
        return pred_rgb, pred_rgb_bg, pred_normals, weights_sum
