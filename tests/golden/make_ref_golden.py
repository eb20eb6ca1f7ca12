"""Generate reference-made golden fixtures (run on a GPU: `python tests/golden/make_ref_golden.py`).

Runs the UNMODIFIED reference CUDA kernels (oracle/_ref/libpsdf_ref_gpu.so, built from the original project's
kernels/permuto_sdf/*GPU.cuh by oracle/ref_shim/Makefile) on small seeded inputs and stores
inputs + outputs in tests/golden/ref_rayops.npz. Packed outputs are canonicalised per ray (the reference hands
out sample slots with an atomic counter, SURVEY.md F8): per-ray counts plus the per-sample arrays concatenated
in ray order. tests/golden/check_golden.py replays the same inputs through the C oracle on the CPU.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import scenes  # noqa: E402
from oracle import ref_gpu as ref  # noqa: E402

V = 32
R = 48


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def N(t):
    return t.detach().cpu().numpy()


def canon(p, names=("z", "dt", "pos", "dirs")):
    se = N(p.start_end)
    n = se[:, 1] - se[:, 0]
    out = {"n": n.astype(np.int32), "fixed_dt": N(p.fixed_dt)}
    for nm in names:
        a = N(getattr(p, nm))
        out[nm] = np.concatenate([a[s:e] for s, e in se] + [a[:0]], 0)
    return out


def put(dst, prefix, d):
    for k, v in d.items():
        dst[prefix + "." + k] = v


def main():
    assert ref.available(), "oracle/_ref/libpsdf_ref_gpu.so missing: run `make -C oracle/ref_shim REF=<checkout of the original project>`"
    G = {}
    o, d = scenes.make_rays(R, seed=11)
    G["in.o"], G["in.d"] = o, d
    to, td = T(o), T(d)
    tr = [0.0, 0.0, 0.0]
    # sphere
    pe, te, px, tx, hit = ref.sphere_ray_intersection(0.5, tr, to, td)
    put(G, "sphere", dict(pe=N(pe), te=N(te), px=N(px), tx=N(tx), hit=N(hit).astype(np.uint8)))
    rng = np.random.RandomState(5)
    phi, ct, u = (rng.rand(64) * 6.28).astype(np.float32), (rng.rand(64) * 2 - 1).astype(np.float32), rng.rand(64).astype(np.float32)
    put(G, "randpts", dict(phi=phi, ct=ct, u=u, out=N(ref.sphere_rand_points_inside(0.5, tr, T(phi), T(ct), T(u)))))
    # grid points + occupancy from the analytic sdf through the reference's update_with_sdf
    pts = ref.occ_grid_points(V, 1.0, tr)
    G["grid.points"] = N(pts)
    G["grid.points_jitter"] = N(ref.occ_grid_points(V, 1.0, tr, None, True))
    idx = rng.randint(0, V ** 3, 500).astype(np.int32)
    G["grid.idx"] = idx
    G["grid.points_subset_jitter"] = N(ref.occ_grid_points(V, 1.0, tr, T(idx), True))
    sdf = scenes.analytic_sdf(N(pts))
    G["grid.sdf"] = sdf
    values = torch.ones(V ** 3, device="cuda"); occ = torch.ones(V ** 3, dtype=torch.bool, device="cuda")
    ref.occ_update_with_sdf(V, 1.0, T(sdf), None, 512.0, 1e-4, values, occ)
    G["grid.occ"] = N(occ).astype(np.uint8)
    v2, o2 = values.clone(), occ.clone()
    s2 = rng.uniform(-0.05, 0.05, (500, 1)).astype(np.float32)
    uidx = np.unique(idx)[:300].astype(np.int32)            # unique: the reference scatter is racy on duplicates
    ref.occ_update_with_sdf(V, 1.0, T(s2[:len(uidx)]), T(uidx), 300.0, 1e-4, v2, o2)
    put(G, "grid.upd_rs", dict(idx=uidx, sdf=s2[:len(uidx)], occ=N(o2).astype(np.uint8), values=N(v2)))
    v3, o3 = torch.ones(V ** 3, device="cuda"), torch.ones(V ** 3, dtype=torch.bool, device="cuda")
    dens = (rng.rand(V ** 3, 1) * 2).astype(np.float32)
    ref.occ_update_with_density(V, T(dens), None, 0.9, 1.2, v3, o3)
    put(G, "grid.upd_density", dict(density=dens, occ=N(o3).astype(np.uint8), values=N(v3)))
    q = rng.uniform(-0.7, 0.7, (2000, 3)).astype(np.float32)
    put(G, "grid.check", dict(pts=q, out=N(ref.occ_check_occupancy(V, 1.0, tr, occ, T(q))).astype(np.uint8)))
    # sampling
    for jitter in (0, 1):
        p = ref.occ_samples_in_occupied_regions(V, 1.0, tr, to, td, te, tx, occ, 2e-3, 24, bool(jitter))
        put(G, "occ_samples.j%d" % jitter, canon(p))
    p0 = ref.occ_samples_in_occupied_regions(V, 1.0, tr, to, td, te, tx, occ, 2e-3, 24, False)
    fs = ref.occ_first_sample_start(V, 1.0, tr, to, td, te, tx, occ)
    put(G, "first_sample", canon(fs))
    adv_pos = (N(td) * 0.1).astype(np.float32)
    np_, nw = ref.occ_advance_to_next_occupied(V, 1.0, tr, td, T(adv_pos), occ)
    put(G, "advance", dict(pos=adv_pos, out=N(np_), within=N(nw).astype(np.uint8)))
    for jitter in (0, 1):
        put(G, "sampler_fg.j%d" % jitter, canon(ref.sampler_fg(to, td, te, tx, 0.5, tr, 0.02, 20, bool(jitter))))
        b = ref.sampler_bg(to, td, tx, 8, 0.5, tr, bool(jitter), False)
        put(G, "sampler_bg.j%d" % jitter, dict(z=N(b.z), dt=N(b.dt), pos=N(b.pos), pos4=N(b.pos4)))
    # volume rendering on the compacted container
    c = p0.compact()
    # canonical (ray ordered) container for the oracle side
    cc = canon(p0)
    Ns = int(cc["n"].sum())
    order = np.concatenate([np.arange(s, e) for s, e in N(c.start_end)] + [np.zeros(0, np.int64)]).astype(np.int64)

    def per_ray(t):          # reference per-sample tensor -> ray-ordered numpy
        return N(t)[order]

    def from_canon(a):       # ray-ordered numpy -> tensor in the reference container's slot order
        out = np.zeros_like(a)
        out[order] = a
        return T(out)
    alpha = rng.uniform(0.8, 1.0, (Ns, 1)).astype(np.float32)
    w = rng.rand(Ns, 1).astype(np.float32)
    rgb = rng.rand(Ns, 3).astype(np.float32)
    G["vr.alpha"], G["vr.w"], G["vr.rgb"] = alpha, w, rgb
    Tt, bg = ref.vr_cumprod(c, from_canon(alpha))
    G["vr.T"], G["vr.bg"] = per_ray(Tt), N(bg)
    G["vr.integrate"] = N(ref.vr_integrate(c, from_canon(rgb), from_canon(w)))
    sr, ss = ref.vr_sum(c, from_canon(w))
    G["vr.sum_ray"], G["vr.sum_sample"] = N(sr), per_ray(ss)
    sr3, _ = ref.vr_sum(c, from_canon(rgb))
    G["vr.sum_ray3"] = N(sr3)
    G["vr.cumsum_f"] = per_ray(ref.vr_cumsum(c, from_canon(w), False))
    G["vr.cumsum_r"] = per_ray(ref.vr_cumsum(c, from_canon(w), True))
    G["vr.cdf"] = per_ray(ref.vr_cdf(c, from_canon(w)))
    G["vr.dt_exit"] = per_ray(ref.vr_compute_dt(c, tx, True))
    sdf_s = scenes.analytic_sdf(cc["pos"])
    G["vr.sdf"] = sdf_s
    G["vr.sdf2alpha"] = per_ray(ref.vr_sdf2alpha(c, from_canon(sdf_s), 512.0, True, 1.0))
    G["vr.sdf2alpha_fixed"] = per_ray(ref.vr_sdf2alpha(c, from_canon(sdf_s), 64.0, False, 2.0))
    gT, gbg = rng.randn(Ns, 1).astype(np.float32), rng.randn(R, 1).astype(np.float32)
    G["vr.gT"], G["vr.gbg"] = gT, gbg
    cs = ref.vr_cumsum(c, from_canon(gT) * Tt, True)
    G["vr.cumprod_bwd"] = per_ray(ref.vr_cumprod_backward(c, from_canon(gT), T(gbg), from_canon(alpha), Tt, bg, cs))
    gp = rng.randn(R, 3).astype(np.float32)
    G["vr.gp"] = gp
    gv, gw = ref.vr_integrate_backward(c, T(gp), from_canon(rgb), from_canon(w), ref.vr_integrate(c, from_canon(rgb), from_canon(w)))
    G["vr.int_bwd_vals"], G["vr.int_bwd_w"] = per_ray(gv), per_ray(gw)
    rad = (rng.rand(Ns, 1) * 200).astype(np.float32)
    G["vr.rad"] = rad
    pr, dp, nbg, nw_ = ref.vr_render_nerf(c, tx, from_canon(rgb), from_canon(rad))
    put(G, "vr.nerf", dict(rgb=N(pr), depth=N(dp), bg=N(nbg), w=per_ray(nw_)))
    # importance resampling round (normalised weights from sdf2alpha)
    a2 = ref.vr_sdf2alpha(c, from_canon(sdf_s), 512.0, True, 1.0).clip(0.0, 1.0)
    T2, _ = ref.vr_cumprod(c, 1 - a2 + 1e-7)
    ww = a2 * T2
    _, wsum = ref.vr_sum(c, ww)
    ww = ww / torch.clamp(wsum, min=1e-6)
    cdf = ref.vr_cdf(c, ww)
    G["imp.cdf"] = per_ray(cdf)
    for jitter in (0, 1):
        q_ = ref.vr_importance_sample(to, td, c, cdf, 8, bool(jitter))
        put(G, "imp.j%d" % jitter, dict(z=N(q_.z), pos=N(q_.pos)))
    q_ = ref.vr_importance_sample(to, td, c, cdf, 8, False)
    c.sdf, c.has_sdf = from_canon(sdf_s), True
    q_.sdf, q_.has_sdf = T(scenes.analytic_sdf(N(q_.pos))), True
    G["imp.sdf"] = N(q_.sdf)
    m = ref.vr_combine(to, td, tx, c, q_)
    put(G, "combine", canon(m, ("z", "dt", "pos", "sdf")))
    # statics
    dirs = rng.randn(257, 3).astype(np.float32); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    G["sh.dirs"] = dirs
    for deg in (1, 3, 5, 7):
        G["sh.deg%d" % deg] = N(ref.spherical_harmonics(T(dirs), deg))
    rgbr, mask, K, tf = scenes.synthetic_reel(nimg=3, H=20, W=24)
    pix = rng.randint(0, 20 * 24, 200).astype(np.int32); img = rng.randint(0, 3, 200).astype(np.int32)
    ro, rd, rgt, rgm = ref.random_rays_from_reel(T(rgbr), T(mask), T(K), T(tf), T(pix), T(img))
    put(G, "reel", dict(pix=pix, img=img, o=N(ro), d=N(rd), gt=N(rgt), gm=N(rgm)))
    out = os.path.join(HERE, "ref_rayops.npz")
    np.savez_compressed(out, **G)
    print("wrote", out, os.path.getsize(out), "bytes,", len(G), "arrays; gpu:", torch.cuda.get_device_name(0))


if __name__ == "__main__":
    main()
