"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

fp64 reference of the differentiable ray-path operations of csrc/volrender.cu (cumprod_alpha2transmittance, integrate_with_weights,
sum_over_each_ray, volume_render_nerf and their backward kernels), in torch float64 over any packed layout: `start_end` with gaps and
skipped rays, or the equal layout. Rays are laid out as a padded, masked [R, L] tensor (neus_fp64.Layout), so every operation is a few
vectorised ops at any ray count; the NeRF render walks the L sample columns, all rays at once.

Semantics, each the kernels' on purpose:
  * a ray is skipped when it is empty or end > max_nr_samples: it has no sample rows, bg_T 1, integrate / sum_ray / pred_rgb / depth 0;
  * T_i = prod_{j<i} a_j over the ray's factors a (already 1 - alpha), bg_T = T_last: the last sample's factor is excluded;
  * the gradients are fp64 autograd of these forwards, except the per-sample broadcast of sum_over_each_ray, whose backward is the
    reference project's pass-through g_vals = g_ray + g_sample (row by row, not the sum of g_sample over the ray);
  * the cumprod backward divides by the factor: it is only the derivative where every factor of the ray is > 1e-6 (`exact_rays`);
  * the NeRF render stops a ray before the first sample whose transmittance T < 1e-4; those and later samples are not written.
    `ambiguous` marks the rays whose fp64 decision is within the error bound of the threshold, where fp32 may decide otherwise.

Error scale A (in units of u = 2^-24): for every output, the sum of the absolute values of the terms rounded along its serial chain,
propagated to first order, as in neus_fp64 / backward_fp64: a chain of k correctly rounded products has A = k (|T| + 2^-126) (gradual underflow); a serial sum (or
fma accumulation) has A = sum of |partial sums|; a product / quotient of rounded operands propagates d_a |b| + d_b |a| (/ b^2).
__expf (the NeRF alpha) has an error of 2 + floor(1.173 |x|) ulp (CUDA programming guide), i.e. 2 (2 + 1.173 |x|) u relative, and
flushes results below 2^-126 to zero. Bounds are first order and worst case, so an observed error stays below u A; EPS = 2^-22 = 4 u
leaves 4x for the second-order terms.
"""
import torch

from oracle.neus_fp64 import TINY, Layout, Tr

F64 = torch.float64
EPS = 2.0 ** -22
FTZ = 2.0 ** -102         # a flushed __expf result: absolute 2^-126 = 2^-102 u
T_STOP = 1e-4             # the NeRF render's early-out (fp32 constant, compared in fp32)
T_STOP32 = float(torch.tensor(T_STOP, dtype=torch.float32))


def layout(start_end, R, max_nr_samples, equal=False, fixed_n=0):
    se = None if equal else torch.as_tensor(start_end).reshape(R, 2)
    return Layout(se, R, max_nr_samples, equal, fixed_n)


def _f64(a):
    return torch.as_tensor(a).detach().to("cpu", F64)


def _col(a):
    """[N] or [N,1] -> [N]"""
    a = _f64(a)
    return a.reshape(a.shape[0]) if a.dim() == 2 and a.shape[1] == 1 else a


def _rows(lay, t, N):
    return lay.scatter(t, N)


def _j(lay):
    return torch.arange(lay.L, dtype=F64)[None, :]


def _rev_cumsum(x):
    return torch.flip(torch.cumsum(torch.flip(x, [1]), 1), [1])


# ------------------------------------------------------------------------------------------------ cumprod
def _cumprod_fwd(lay, a):
    bb = torch.where(lay.valid & ~lay.last, a, torch.ones_like(a))
    T = torch.cumprod(torch.cat([torch.ones_like(bb[:, :1]), bb[:, :-1]], 1), 1)
    T = torch.where(lay.valid, T, torch.zeros_like(T))
    return T, torch.prod(bb, 1)


def cumprod(lay, alpha):
    """T [N] (rows of computed rays), bg [R], and their error scales"""
    a = lay.gather(_col(alpha))
    N = _col(alpha).shape[0]
    T, bg = _cumprod_fwd(lay, a)
    A_T = _j(lay) * (T.abs() + TINY)
    A_bg = (lay.n.to(F64) - 1).clamp(min=0) * (bg.abs() + TINY)
    T_r, rows = _rows(lay, T, N)
    return dict(T=T_r, A_T=_rows(lay, A_T, N)[0], rows=rows, bg=bg, A_bg=A_bg)


def cumprod_backward(lay, alpha, g_T, g_bg):
    """d/d alpha of sum(g_T T) + sum(g_bg bg_T), for the kernel chain T (cumprod) -> cumsumLV = reverse cumsum of g_T * T ->
    cumprod_backward(g_bg, alpha, bg_T, cumsumLV). `exact_rays`: rays where the division form is the derivative."""
    N = _col(alpha).shape[0]
    a = lay.gather(_col(alpha)).requires_grad_(True)
    gT, gbg = lay.gather(_col(g_T)), _col(g_bg)
    T, bg = _cumprod_fwd(lay, a)
    (ga,) = torch.autograd.grad((gT * T).sum() + (gbg * bg).sum(), a)
    with torch.no_grad():
        j = _j(lay)
        lv = gT * T
        A_lv = (j + 1) * (lv.abs() + TINY)
        cs = _rev_cumsum(lv)
        A_cs = _rev_cumsum(A_lv) + _rev_cumsum(cs.abs())
        nxt = lambda x: torch.cat([x[:, 1:], torch.zeros_like(x[:, :1])], 1)
        active = lay.valid & ~lay.last
        ad = a.detach().abs().clamp(min=1e-30)
        gb = (gbg * bg).abs()[:, None]
        q1, q2 = nxt(cs).abs() / ad, gb / ad
        A = (nxt(A_cs) / ad + q1) + (lay.n.to(F64)[:, None] * (gb + TINY) / ad + q2) + ga.abs() + 2 * TINY
        A = torch.where(active, A, torch.zeros_like(A))
        exact = ~((a.detach() <= 1e-6) & active).any(1)
    ga_r, rows = _rows(lay, ga, N)
    return dict(g_alpha=ga_r, A=_rows(lay, A, N)[0], rows=rows, exact_rays=exact)


# ------------------------------------------------------------------------------------------------ integrate
def integrate(lay, vals, w):
    v, ww = lay.gather(_f64(vals)), lay.gather(_col(w))
    p = torch.cumsum(ww[..., None] * v, 1)
    return dict(out=p[:, -1], A=p.abs().sum(1))


def integrate_backward(lay, g_pred, vals, w):
    """d/d(vals, w) of sum(g_pred * integrate(vals, w)); the three-channel derivative (not the reference_bugs formula)"""
    N = _f64(vals).shape[0]
    v = lay.gather(_f64(vals)).requires_grad_(True)
    ww = lay.gather(_col(w)).requires_grad_(True)
    g = _f64(g_pred)
    gv, gw = torch.autograd.grad((g[:, None, :] * (ww[..., None] * v)).sum(), (v, ww))
    with torch.no_grad():
        v, ww = v.detach(), ww.detach()
        A_gv = gv.abs()
        t1 = (g[:, None, 1] * v[..., 1]).abs()
        t2 = (g[:, None, 0] * v[..., 0] + g[:, None, 1] * v[..., 1]).abs()
        A_gw = t1 + t2 + gw.abs()
    gv_r, rows = _rows(lay, gv, N)
    return dict(g_vals=gv_r, A_vals=_rows(lay, A_gv, N)[0], g_w=_rows(lay, gw, N)[0], A_w=_rows(lay, A_gw, N)[0], rows=rows)


# ------------------------------------------------------------------------------------------------ sum over each ray
def sum_over_each_ray(lay, vals):
    vals = _f64(vals)
    N, D = vals.shape
    v = lay.gather(vals)
    p = torch.cumsum(v, 1)
    s, A = p[:, -1], p.abs().sum(1)
    bs = torch.where(lay.valid[..., None], s[:, None, :].expand(-1, lay.L, -1), torch.zeros_like(v))
    bA = torch.where(lay.valid[..., None], A[:, None, :].expand(-1, lay.L, -1), torch.zeros_like(v))
    ss, rows = _rows(lay, bs, N)
    return dict(sum_ray=s, A_ray=A, sum_sample=ss, A_sample=_rows(lay, bA, N)[0], rows=rows)


def sum_over_each_ray_backward(lay, g_ray, g_sample):
    """fp64 autograd of sum(g_ray * sum_ray), plus the pass-through of g_sample (see the module docstring)"""
    g_sample = _f64(g_sample)
    N, D = g_sample.shape
    v = torch.zeros(lay.R, lay.L, D, dtype=F64, requires_grad=True)
    s = torch.where(lay.valid[..., None], v, torch.zeros_like(v)).sum(1)
    (g,) = torch.autograd.grad((_f64(g_ray) * s).sum(), v)
    g = torch.where(lay.valid[..., None], g + lay.gather(g_sample), torch.zeros_like(g))
    g_r, rows = _rows(lay, g, N)
    return dict(g_vals=g_r, A=g_r.abs(), rows=rows)


# ------------------------------------------------------------------------------------------------ NeRF render
def _expf(x):
    """__expf of a tracked argument"""
    e = torch.exp(x.v)
    k = 2.0 * (2.0 + 1.173 * x.v.abs())
    return Tr(e, e * x.d + k * e + FTZ)


def volume_render_nerf(lay, rgb, radiance, z, dt, g_pred=None, g_bg=None):
    """forward (pred_rgb [R,3], depth [R], bg_T [R], w [N] on `written` rows) and, with g_pred / g_bg, the fp64 gradient of
    sum(g_pred pred_rgb) + sum(g_bg bg_T) w.r.t. rgb and radiance at fixed stop points. Error scales A_* for all of them; the
    backward's scale follows the kernel's formula, which reads the forward's pred_rgb and bg_T (their errors included)."""
    rgb = _f64(rgb)
    N = rgb.shape[0]
    c = lay.gather(rgb).requires_grad_(True)
    sg = lay.gather(_col(radiance)).requires_grad_(True)
    zz, dd = lay.gather(_col(z)), lay.gather(_col(dt))
    R, L = lay.R, lay.L
    # fp64 values, and the stop decision: sample i is used iff T_i >= 1e-4 for the T before it (T is non-increasing)
    x = -(sg * dd)
    al = 1.0 - torch.exp(x)
    b = torch.exp(x)
    T = torch.cumprod(torch.cat([torch.ones_like(b[:, :1]), b[:, :-1]], 1), 1)
    used = lay.valid & (T.detach() >= T_STOP32)
    wv = torch.where(used, al * T, torch.zeros_like(T))
    pred = (wv[..., None] * c).sum(1)
    depth = (wv * zz).sum(1)
    bg = torch.where(lay.skip, torch.ones_like(T[:, 0]), torch.prod(torch.where(used, b, torch.ones_like(b)), 1))
    out = dict(pred=pred.detach(), depth=depth.detach(), bg=bg.detach())
    if g_pred is not None:
        gp, gb = _f64(g_pred), _col(g_bg)
        g_c, g_s = torch.autograd.grad((gp * pred).sum() + (gb * bg).sum(), (c, sg))
        out["g_rgb"] = _rows(lay, torch.where(used[..., None], g_c, torch.zeros_like(g_c)), N)[0]
        out["g_rad"] = _rows(lay, torch.where(used, g_s, torch.zeros_like(g_s)), N)[0]
    # error scales: the kernel's chain, tracked column by column for all rays at once
    with torch.no_grad():
        c, sg = c.detach(), sg.detach()
        Tt = Tr(torch.ones(R, dtype=F64))
        acc = [Tr(torch.zeros(R, dtype=F64)) for _ in range(3)]
        dep = Tr(torch.zeros(R, dtype=F64))
        A_w = torch.zeros(R, L, dtype=F64)
        A_Tcol = torch.zeros(R, L, dtype=F64)
        amb = torch.zeros(R, dtype=torch.bool)
        cols = []
        for i in range(L):
            u = used[:, i]
            near = lay.valid[:, i] & ((Tt.v - T_STOP32).abs() <= 2 * EPS * Tt.d + 1e-12)
            amb |= near
            xi = Tr(-sg[:, i] * dd[:, i], (sg[:, i] * dd[:, i]).abs())
            e = _expf(xi)
            a = 1.0 - e
            w = a * Tt
            A_w[:, i] = w.d
            new = [Tr(w.v * c[:, i, k] + acc[k].v, w.d * c[:, i, k].abs() + acc[k].d + (w.v * c[:, i, k] + acc[k].v).abs()) for k in range(3)]
            nd = Tr(w.v * zz[:, i] + dep.v, w.d * zz[:, i].abs() + dep.d + (w.v * zz[:, i] + dep.v).abs())
            Tn = Tt * (1.0 - a)
            cols.append((w, Tn, a, [n for n in new]))
            acc = [n.where(u, o) for n, o in zip(new, acc)]
            dep = nd.where(u, dep)
            Tt = Tn.where(u, Tt)
            A_Tcol[:, i] = Tt.d
        out.update(A_pred=torch.stack([a_.d for a_ in acc], 1), A_depth=dep.d, A_bg=torch.where(lay.skip, torch.zeros_like(Tt.d), Tt.d))
        out["w"], out["written"] = _rows(lay, torch.where(used, wv.detach(), torch.zeros_like(wv)), N)
        out["written"] = _rows(lay, used.to(F64), N)[0] > 0
        out["A_w"] = _rows(lay, torch.where(used, A_w, torch.zeros_like(A_w)), N)[0]
        out["ambiguous"] = amb & ~lay.skip
        if g_pred is not None:
            fx = [Tr(pred[:, k].detach(), out["A_pred"][:, k]) for k in range(3)]
            lastT = Tr(bg.detach(), out["A_bg"])
            A_g = torch.zeros(R, L, dtype=F64)
            A_gc = torch.zeros(R, L, 3, dtype=F64)
            for i in range(L):
                w, Tn, a, up = cols[i]
                dtk = Tr(dd[:, i])
                grad = Tr(torch.zeros(R, dtype=F64))
                for k in range(3):
                    gk = Tr(gp[:, k])
                    grad = grad + (gk * dtk) * (Tn * Tr(c[:, i, k]) - (fx[k] - up[k]))
                    A_gc[:, i, k] = (gk * w).d
                grad = grad + Tr(gb) * (Tr(-dd[:, i]) * lastT)
                A_g[:, i] = grad.d
            out["A_g_rad"] = _rows(lay, torch.where(used, A_g, torch.zeros_like(A_g)), N)[0]
            out["A_g_rgb"] = _rows(lay, torch.where(used[..., None], A_gc, torch.zeros_like(A_gc)), N)[0]
    return out


# ------------------------------------------------------------------------------------------------ comparison
def check(name, got, ref, A, mask=None, report=None):
    """max|err| / max|ref| <= 1e-3 and |err| <= EPS A element by element (over `mask`); returns the worst err / bound ratio"""
    got, ref, A = torch.broadcast_tensors(_f64(got), _f64(ref), _f64(A))
    if mask is not None:
        m = torch.as_tensor(mask).to(torch.bool)
        while m.dim() < got.dim():
            m = m[..., None]
        m = m.expand_as(got)
        got, ref, A = got[m], ref[m], A[m]
    if got.numel() == 0:
        return 0.0
    assert torch.isfinite(got).all(), "%s: non-finite values" % name
    err = (got - ref).abs()
    scale = ref.abs().max()
    rel = float(err.max() / scale) if scale > 0 else float(err.max())
    assert rel <= 1e-3, "%s: max|err| / max|ref| = %.3g > 1e-3" % (name, rel)
    bound = EPS * A
    ratio = float((err / bound.clamp(min=1e-300)).max())
    bad = err > bound
    assert not bool(bad.any()), "%s: %d elements above EPS*A, worst err/bound %.3g" % (name, int(bad.sum()), ratio)
    if report is not None:
        report[name] = max(report.get(name, 0.0), ratio)
    return ratio


# ------------------------------------------------------------------------------------------------ layouts
RAGGED_LENGTHS = (0, 1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 128, 1023)


def ragged_layout(seed, copies=2, lengths=RAGGED_LENGTHS, n_skip=4):
    """start_end [R,2] int32 of a ragged packed set: every length `copies` times in random order, random gaps between rays, and
    `n_skip` rays interleaved whose end lies past max_nr_samples (skipped by every kernel). Returns (start_end, max_nr_samples)."""
    import numpy as np
    rng = np.random.RandomState(seed)
    ls = np.array(list(lengths) * copies)
    rng.shuffle(ls)
    se, cur = [], 0
    for n in ls:
        cur += int(rng.randint(0, 4))
        se.append((cur, cur + int(n)))
        cur += int(n)
    M = cur + int(rng.randint(0, 3))
    for _ in range(n_skip):
        s = int(rng.randint(0, M))
        se.insert(int(rng.randint(0, len(se) + 1)), (s, M + 1 + int(rng.randint(0, 40))))
    return np.asarray(se, np.int32), M


def ray_of_row(lay, N):
    """ray index of every sample row of a computed ray, -1 for the rows no computed ray owns"""
    import numpy as np
    out = np.full(N, -1, np.int64)
    idx, valid = lay.idx.numpy(), lay.valid.numpy()
    out[idx[valid]] = np.broadcast_to(np.arange(lay.R)[:, None], idx.shape)[valid]
    return out


def rows_of(lay, N, ray_mask):
    """[N] bool: the sample rows of the computed rays selected by `ray_mask` [R]"""
    r = torch.as_tensor(ray_of_row(lay, N))
    return (r >= 0) & torch.as_tensor(ray_mask)[r.clamp(min=0)]
