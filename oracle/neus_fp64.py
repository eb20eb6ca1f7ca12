"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

fp64 reference of the NeuS loss head (csrc/neus_fused.cu: compositing, colour head, per-ray loss terms and their backward) and of the
scalar loss terms (csrc/iter_glue.cu psdf_loss_terms), in torch float64 with autograd. Rays are laid out as a padded, masked [R, Lmax]
tensor, so that the graph is a few dozen ops at any ray count.

Semantics (the reference project's VolumeRenderingNeus.compute_weights / integrate and the losses of train_permuto_sdf.py), each on purpose:
  * inv_s is clipped to [1e-6, 1e6]; the gradient passes only inside that range, ends included (torch.clamp);
  * true_cos = dir . g, iter_cos = -(relu(.5 - .5 c)(1 - r) + relu(-c) r), with torch's relu gradient of 0 at the kink;
  * prev / next = sdf -/+ iter_cos dt / 2, alpha = clip((sig(prev s) - sig(next s) + 1e-5) / (sig(prev s) + 1e-5), 0, 1), formed as
    1 - sig(next s) / (sig(prev s) + 1e-5) so that its fp64 derivative does not cancel at saturation;
  * T_i = prod_{j<i} (1 - alpha_j + 1e-7) and bg_T = T_last: the last sample's factor is excluded;
  * the cumprod backward divides by max(1 - alpha + 1e-7, 1e-6) (ClampedCumprod): the reference kernel's clamp_min(alpha_cur, 1e-6)
    on the factor, not the true derivative where the factor is below 1e-6;
  * the integrate backward is the correct three-channel one (not the reference kernel's green-channel bug, `reference_bugs`);
  * L1 on pred after the background blend, sign(0) = 0, times the hit weight;
  * BCE on clip(w_sum, 1e-3, 1 - 1e-3) with the bounds rounded to fp32 (as the reference's fp32 torch rounds them: -log(1 - p) at
    the upper bound is 1.3e-5 relative away from the fp64 constant's), the log clamped at -100;
  * eikonal (|g| - 1)^2 with a zero gradient at g = 0 (torch's norm backward);
  * colour head sigmoid(x (1 + wd[img]) + b[img]), identity at img == fixed_img (and without img_idx or weight_delta);
  * curvature acos(clamp(n . n_s, -1 + 1e-6, 1 - 1e-6)) / pi with F.normalize (eps 1e-12);
  * empty rays and rays with end > max_nr_samples are skipped: no sample rows, w_sum 0, bg_T 1, pred = the background (or 0);
  * psdf_loss_terms: sums of the per-ray terms, means over the valid rows (or the data-parallel mean count), the off-surface term
    w_off mean(exp(-100 |s|)) with its seed, w_lip prod softplus(c_l) (softplus threshold 20).

The backward reference is evaluated at the forward values the backward kernel reads (saved alpha, pred, w_sum, bg_T): their values are
substituted by straight-through terms, the gradient is the fp64 one. So the L1 sign at pred == gt and the BCE clip decide as the kernel
does, and the clamped cumprod divisor is formed from the saved alpha, exactly as in the kernel.

Error scale A (`Tr`, tracked arithmetic): every kernel expression is re-evaluated in fp64 carrying, beside its value v, the linearised
propagation of absolute rounding terms d, in units of u = 2^-24: a correctly rounded fp32 operation adds |v| (half an ulp is at most
u |v|, plus 2^-150 = 2^-126 u of gradual underflow for a product or quotient); a product / quotient propagates d_a |b| + d_b |a| (/ b^2); a function f propagates |f'| d_x and adds k |f(x)|, k = 4 for expf and
acosf (2 ulp), 2 for logf (1 ulp), 1 for sqrtf. __expf (the kernels' sigmoid in the alpha) has an error of 2 + floor(1.173 |x|) ulp (CUDA
programming guide), k = 2 (2 + 1.173 |x|): ~200 u at |x| ~ 88, where saturation takes it. The cancellations in pc - nc, 1 - pc,
1 - alpha and gpc + gnc are carried by d: their operands' absolute errors survive while the value shrinks. Serial sums add the absolute
value of every partial sum; tree / atomic sums |sum of terms| times the depth. Bounds are first order and worst case (every rounding
with the worst sign), so an observed error stays below u A; EPS = 2^-22 = 4 u leaves 4x for the second-order terms and the freedom
of fma contraction. tests/test_neus_loss_fp64_reference_cpu.py checks it against an fp32 emulation of the kernels' arithmetic with the
__expf error injected at its documented bound.
"""
import math

import torch
import torch.nn.functional as F

F64 = torch.float64
EPS = 2.0 ** -22
INV_PI = 0.3183098861837907
P_LO, P_HI = float(torch.tensor(1e-3)), float(torch.tensor(1.0 - 1e-3))     # the BCE clip as fp32 constants (torch rounds them so too)
TINY = 2.0 ** -126        # gradual underflow: a product or quotient may round by half the smallest subnormal, 2^-150 = 2^-126 u


# ------------------------------------------------------------------------------------------------ ray layout
class Layout:
    """padded [R, L] view of a packed sample set: idx (row of each slot, 0 where unused), valid [R, L], n [R], skip [R]"""

    def __init__(self, start_end, R, max_nr_samples, equal=False, fixed_n=0, device="cpu"):
        if equal:
            start = torch.arange(R, dtype=torch.long) * fixed_n
            end = start + fixed_n
        else:
            se = start_end.detach().cpu().long().reshape(R, 2)
            start, end = se[:, 0], se[:, 1]
        n = end - start
        self.R, self.start, self.end, self.n = R, start, end, n
        self.skip = (end > max_nr_samples) | (n == 0)
        self.L = max(int(n[~self.skip].max()) if bool((~self.skip).any()) else 1, 1)
        j = torch.arange(self.L)
        self.valid = (j[None, :] < n[:, None]) & ~self.skip[:, None]
        self.idx = torch.where(self.valid, start[:, None] + j[None, :], torch.zeros_like(self.valid, dtype=torch.long))
        self.last = self.valid & (j[None, :] == (n[:, None] - 1))     # the last sample of every computed ray
        self.chunks = torch.clamp((n + 31) // 32, min=1)
        self.device = device
        self.idx, self.valid, self.last = self.idx.to(device), self.valid.to(device), self.last.to(device)

    def gather(self, t):
        """[N, ...] -> [R, L, ...], zero in unused slots"""
        g = t[self.idx.reshape(-1)].reshape(self.R, self.L, *t.shape[1:])
        m = self.valid.reshape(self.R, self.L, *([1] * (t.dim() - 1)))
        return torch.where(m, g, torch.zeros_like(g))

    def scatter(self, t, N):
        """[R, L, ...] -> [N, ...] rows of the computed rays (the rest zero) and the mask of those rows"""
        out = torch.zeros((N,) + tuple(t.shape[2:]), dtype=t.dtype, device=t.device)
        m = self.valid.reshape(-1)
        out[self.idx.reshape(-1)[m]] = t.reshape(self.R * self.L, *t.shape[2:])[m]
        rows = torch.zeros(N, dtype=torch.bool, device=t.device)
        rows[self.idx.reshape(-1)[m]] = True
        return out, rows


class ClampedCumprod(torch.autograd.Function):
    """T_i = prod_{j<i} b_j over the valid slots, bg_T = T of the last sample; backward divides by max(b, 1e-6)"""

    @staticmethod
    def forward(ctx, b, valid, last):
        bb = torch.where(valid & ~last, b, torch.ones_like(b))
        T = torch.cumprod(torch.cat([torch.ones_like(bb[:, :1]), bb[:, :-1]], 1), 1)
        T = torch.where(valid, T, torch.zeros_like(T))
        bgT = torch.cumprod(bb, 1)[:, -1]
        ctx.save_for_backward(b, T, bgT, valid, last)
        return T, bgT

    @staticmethod
    def backward(ctx, gT, gbg):
        b, T, bgT, valid, last = ctx.saved_tensors
        lv = gT * T
        suffix = torch.flip(torch.cumsum(torch.flip(lv, [1]), 1), [1]) - lv           # sum_{k>i} gT_k T_k
        active = valid & ~last
        gb = torch.where(active, (suffix + (gbg * bgT)[:, None]) / torch.clamp(b, min=1e-6), torch.zeros_like(b))
        return gb, None, None


def _st(x, value):
    """x with its value replaced by `value` (straight through: the gradient is x's)"""
    return x if value is None else x + (value.to(x) - x).detach()


# ------------------------------------------------------------------------------------------------ inputs
class NeusInputs:
    """the arguments of one psdf_neus_* call (CPU or CUDA tensors, fp32 / int as the kernels take them)"""

    def __init__(self, start_end, R, N, max_nr_samples, sdf, grad, rgb, dirs, dt, inv_s, cos_anneal, gt_rgb=None, gt_mask=None, hit=None,
                 bg_rgb=None, head=False, img_idx=None, weight_delta=None, bias=None, fixed_img=-1, gs=None, equal=False, fixed_n=0):
        self.__dict__.update(locals())
        del self.__dict__["self"]


def _f64(t):
    return None if t is None else t.detach().to(F64)


def forward_reference(I, saved=None, device="cpu", leaves=False):
    """fp64 forward of the NeuS loss head. Returns a dict: alpha, T, w [N] (rows of computed rays; `rows` marks them), pred [R,3],
    wsum, bgT [R], ray_loss [R,3], eik [R, L], curv [R, L] (with gs), normals [R,3], pred_bg [R,3] (with bg_rgb), and the leaves when
    asked (for autograd). `saved` = dict(alpha [N], pred [R,3], wsum [R], bgT [R]) substitutes the kernel's values (see the docstring)."""
    lay = Layout(I.start_end, I.R, I.max_nr_samples, I.equal, I.fixed_n, device)
    leaf = lambda t: t.detach().requires_grad_(True) if leaves else t
    lv = {k: leaf(_f64(getattr(I, k)).to(device)) for k in ("sdf", "grad", "rgb")}
    lv["inv_s"] = leaf(_f64(I.inv_s).to(device).reshape(-1)[:1])
    if I.bg_rgb is not None:
        lv["bg_rgb"] = leaf(_f64(I.bg_rgb).to(device))
    use_cal = I.head and I.img_idx is not None and I.weight_delta is not None
    if use_cal:
        lv["wd"] = leaf(_f64(I.weight_delta).to(device))
        lv["bias"] = leaf(_f64(I.bias if I.bias is not None else torch.zeros_like(I.weight_delta)).to(device))
    if I.gs is not None:
        lv["gs"] = leaf(_f64(I.gs).to(device))
    dirs, dt = _f64(I.dirs).to(device), _f64(I.dt).to(device).reshape(-1)
    s = torch.clamp(lv["inv_s"], 1e-6, 1e6)
    r = float(I.cos_anneal)
    sdf, g, d, dtt = lay.gather(lv["sdf"].reshape(-1)), lay.gather(lv["grad"]), lay.gather(dirs), lay.gather(dt)
    tc = (d * g).sum(-1)
    ic = -(F.relu(-tc * 0.5 + 0.5) * (1.0 - r) + F.relu(-tc) * r)
    nxt, prv = sdf + ic * dtt * 0.5, sdf - ic * dtt * 0.5
    pc, nc = torch.sigmoid(prv * s), torch.sigmoid(nxt * s)
    # (pc - nc + 1e-5) / (pc + 1e-5) written as 1 - nc / (pc + 1e-5): the same value, but autograd then forms d/dpc as
    # nc / (pc + 1e-5)^2 (as the kernels do) instead of 1/(pc + 1e-5) - q/(pc + 1e-5), whose two ~1e5 terms cancel to ~1e-11 of
    # fp64 noise where the true value is ~nc 1e10 (~1e-26 at saturation)
    alpha = (1.0 - nc / (pc + 1e-5)).clamp(0.0, 1.0)
    if saved is not None:
        alpha = _st(alpha, lay.gather(saved["alpha"].detach().to(device).reshape(-1)))
    valid = lay.valid
    alpha = torch.where(valid, alpha, torch.zeros_like(alpha))
    T, bgT = ClampedCumprod.apply(1.0 - alpha + 1e-7, valid, lay.last)
    w = alpha * T
    x = lay.gather(lv["rgb"])
    if I.head:
        if use_cal:
            img = I.img_idx.detach().to(device).long().reshape(-1)
            cal = (img != int(I.fixed_img)).to(F64)[:, None]
            hw = 1.0 + lv["wd"][img] * cal
            hb = lv["bias"][img] * cal
            c = torch.sigmoid(x * hw[:, None, :] + hb[:, None, :])
        else:
            c = torch.sigmoid(x)
    else:
        c = x
    pred = (w[..., None] * c).sum(1)
    if saved is not None:
        bgT = _st(bgT, saved["bgT"].detach().to(device).reshape(-1))
    pred_bg = None
    if I.bg_rgb is not None:
        pred_bg = bgT[:, None] * lv["bg_rgb"]
        pred = pred + pred_bg
    wsum = w.sum(1)
    if saved is not None:
        pred = _st(pred, saved["pred"].detach().to(device).reshape(-1, 3))
        wsum = _st(wsum, saved["wsum"].detach().to(device).reshape(-1))
    out = dict(layout=lay, pred=pred, wsum=wsum, bgT=bgT, pred_bg=pred_bg, pc=pc, nc=nc, s=s, lv=lv)
    nw = (w[..., None] * g).sum(1)
    out["normals"] = F.normalize(nw, dim=1, eps=1e-12)
    N = I.sdf.reshape(-1).shape[0]
    out["alpha"], out["rows"] = lay.scatter(alpha, N)
    out["T"], _ = lay.scatter(T, N)
    out["w"], _ = lay.scatter(w, N)
    out["alpha_pad"], out["T_pad"], out["w_pad"], out["c_pad"] = alpha, T, w, c
    # per-ray loss terms
    h = torch.ones(I.R, dtype=F64, device=device) if I.hit is None else (I.hit.detach().to(device).reshape(-1) != 0).to(F64)
    gt = _f64(I.gt_rgb).to(device) if I.gt_rgb is not None else torch.zeros_like(pred)
    l1 = (gt - pred).abs().sum(1) * h
    if I.gt_mask is not None:
        m = _f64(I.gt_mask).to(device).reshape(-1)
        p = wsum.clamp(P_LO, P_HI)
        bce = -(m * torch.clamp(torch.log(p), min=-100.0) + (1.0 - m) * torch.clamp(torch.log(1.0 - p), min=-100.0))
    else:
        bce = torch.zeros_like(l1)
    nrm = torch.linalg.vector_norm(g, dim=-1)
    eik = torch.where(valid, (nrm - 1.0) ** 2, torch.zeros_like(nrm))
    out["eik"] = eik
    out["ray_loss"] = torch.stack([l1, bce, eik.sum(1)], 1)
    if I.gs is not None:
        gsp = lay.gather(lv["gs"])
        dot = (F.normalize(g, dim=-1, eps=1e-12) * F.normalize(gsp, dim=-1, eps=1e-12)).sum(-1)
        curv = torch.acos(dot.clamp(-1.0 + 1e-6, 1.0 - 1e-6)) / math.pi
        out["curv"] = torch.where(valid, curv, torch.zeros_like(curv))
    return out


def head_loss(out, scale_rgb, scale_mask, scale_eik, curv_k=0.0, gtot=1.0):
    """the scalar the backward kernels differentiate: gtot (scale_rgb sum L1 + scale_mask sum BCE + scale_eik sum eik + curv_k sum curv)"""
    rl = out["ray_loss"]
    loss = scale_rgb * rl[:, 0].sum() + scale_mask * rl[:, 1].sum() + scale_eik * out["eik"].sum()
    if "curv" in out and curv_k != 0.0:
        loss = loss + curv_k * out["curv"].sum()
    return gtot * loss


def backward_reference(I, saved, scale_rgb, scale_mask, scale_eik, curv_k=0.0, gtot=1.0, device="cpu"):
    """d head_loss / d {sdf, grad, rgb (raw x with the head), bg_rgb, inv_s, weight_delta, bias, gs} at the saved forward values"""
    out = forward_reference(I, saved, device, leaves=True)
    loss = head_loss(out, scale_rgb, scale_mask, scale_eik, curv_k, gtot)
    keys = [k for k in ("sdf", "grad", "rgb", "bg_rgb", "inv_s", "wd", "bias", "gs") if k in out["lv"]]
    gr = torch.autograd.grad(loss, [out["lv"][k] for k in keys], allow_unused=True)
    res = {k: (torch.zeros_like(out["lv"][k]) if g is None else g) for k, g in zip(keys, gr)}
    res["rows"] = out["rows"]
    return res


# ------------------------------------------------------------------------------------------------ tracked arithmetic (error scales)
class Tr:
    """a value and its absolute rounding-error scale in units of u = 2^-24 (see the module docstring)"""
    __slots__ = ("v", "d")

    def __init__(self, v, d=None):
        self.v = v if isinstance(v, torch.Tensor) else torch.tensor(float(v), dtype=F64)
        self.d = torch.zeros_like(self.v) if d is None else d

    def __add__(self, o):
        o = o if isinstance(o, Tr) else Tr(o)
        v = self.v + o.v
        return Tr(v, self.d + o.d + v.abs())

    def __radd__(self, o):
        return self.__add__(o)

    def __sub__(self, o):
        o = o if isinstance(o, Tr) else Tr(o)
        v = self.v - o.v
        return Tr(v, self.d + o.d + v.abs())

    def __rsub__(self, o):
        return Tr(o) - self

    def __neg__(self):
        return Tr(-self.v, self.d)

    def __mul__(self, o):
        o = o if isinstance(o, Tr) else Tr(o)
        v = self.v * o.v
        return Tr(v, self.d * o.v.abs() + o.d * self.v.abs() + v.abs() + TINY)

    def __rmul__(self, o):
        return self.__mul__(o)

    def __truediv__(self, o):
        o = o if isinstance(o, Tr) else Tr(o)
        v = self.v / o.v
        return Tr(v, self.d / o.v.abs() + o.d * (v / o.v).abs() + v.abs() + TINY)

    def __rtruediv__(self, o):
        return Tr(o) / self

    def exact(self):
        """a result known to be exact (no rounding of its own), e.g. a product with 0.5"""
        return self

    def where(self, m, other):
        other = other if isinstance(other, Tr) else Tr(torch.full_like(self.v, float(other)))
        return Tr(torch.where(m, self.v, other.v), torch.where(m, self.d, other.d))


def tr_exact(v):
    return Tr(v.to(F64))


def tr_scale(t, c):
    """t * c for a power of two c: exact"""
    return Tr(t.v * c, t.d * abs(c))


def tr_clamp(t, lo=None, hi=None):
    v = t.v
    if lo is not None:
        v = torch.clamp(v, min=lo)
    if hi is not None:
        v = torch.clamp(v, max=hi)
    inside = v == t.v
    return Tr(v, torch.where(inside, t.d, torch.zeros_like(t.d)))


def tr_fn(x, f, df, k):
    v = f(x.v)
    return Tr(v, df(x.v).abs() * x.d + k * v.abs())


def _tr_sigmoid(x, k):
    """1 / (1 + e), e = exp(-x) with a relative error of k u: d = pc (1 - pc) (d_x + k) + 2 pc (the sum and the quotient), in the
    overflow-free form (e = inf gives pc = 0 in the kernels and here)"""
    v = torch.sigmoid(x.v)
    d = v * (1.0 - v) * (x.d + k) + 2.0 * v + TINY
    # past exp's fp32 range (|x| > 88.72) e is inf and the kernels' result 0: all of v is error
    return Tr(v, torch.where(-x.v > 88.72, d + v * 2.0 ** 24, d))


def tr_sigmoid_fast(x):
    """1 / (1 + __expf(-x)): __expf has 2 + floor(1.173 |x|) ulp, at most 2 u each"""
    return _tr_sigmoid(x, 2.0 * (2.0 + torch.floor(1.173 * x.v.abs())))


def tr_sigmoid_exact(x):
    """1 / (1 + expf(-x)), expf 2 ulp"""
    return _tr_sigmoid(x, 4.0)


def tr_sqrt(x):
    """sqrtf (correctly rounded); an error d of x moves sqrt(x) by at most min(d / (2 sqrt x), sqrt(d u)) (the second near x = 0)"""
    v = torch.sqrt(x.v)
    prop = torch.minimum(x.d * 0.5 / torch.clamp(v, min=1e-300), torch.sqrt(x.d) * 2.0 ** 12)
    return Tr(v, prop + v.abs())


def tr_serial_sum(terms, dim):
    """a left-to-right running sum along dim: sum of the terms' d and of every |partial sum|"""
    part = torch.cumsum(terms.v, dim)
    return Tr(terms.v.sum(dim), terms.d.sum(dim) + part.abs().sum(dim))


def tr_suffix(terms):
    """S_i = sum_{k>i} terms_k, accumulated from the end one term at a time (the backward's reverse sweep)"""
    rev = torch.flip(torch.cumsum(torch.flip(terms.v, [1]), 1), [1])         # sum_{k>=i}
    S = rev - terms.v
    dd = torch.flip(torch.cumsum(torch.flip(terms.d + rev.abs(), [1]), 1), [1]) - (terms.d + rev.abs())
    return Tr(S, dd)


def _tr_dot3(a, b):
    """a0 b0 + a1 b1 + a2 b2 over the last dim, separately rounded"""
    p = [Tr(a.v[..., k], a.d[..., k]) * Tr(b.v[..., k], b.d[..., k]) for k in range(3)]
    return (p[0] + p[1]) + p[2]


def _tr_normalize3(x):
    """normalize3n of neus_fused.cu / F.normalize(eps 1e-12): (unit vector, 1 / den, ok)"""
    n = tr_sqrt(_tr_dot3(x, x))
    ok = n.v > 1e-12
    den = tr_clamp(n, lo=1e-12)
    comps = [Tr(x.v[..., k], x.d[..., k]) / den for k in range(3)]
    return comps, 1.0 / den, ok


def _col(t, k):
    return Tr(t.v[..., k], t.d[..., k])


def error_scales(I, fwd_saved=None, scale_rgb=0.0, scale_mask=0.0, scale_eik=0.0, curv_k=0.0, gtot=1.0, det_rays_per_img=None,
                 device="cpu"):
    """error scales A of every forward output (fwd_saved None) or backward output (fwd_saved = the kernel's forward values), following
    the kernels' expression order. Returns per-output A tensors in the layout of the outputs ([N], [N,3], [R], [R,3], [1], [imgs,3])."""
    lay = Layout(I.start_end, I.R, I.max_nr_samples, I.equal, I.fixed_n, device)
    N = I.sdf.reshape(-1).shape[0]
    s_val = torch.clamp(_f64(I.inv_s).to(device).reshape(-1)[:1], 1e-6, 1e6)
    s = Tr(s_val.expand(lay.R, lay.L).clone())
    r = float(I.cos_anneal)
    r32 = float(torch.tensor(r, dtype=torch.float32))
    sdf = tr_exact(lay.gather(_f64(I.sdf).to(device).reshape(-1)))
    g = tr_exact(lay.gather(_f64(I.grad).to(device)))
    dv = tr_exact(lay.gather(_f64(I.dirs).to(device)))
    dt = tr_exact(lay.gather(_f64(I.dt).to(device).reshape(-1)))
    x = tr_exact(lay.gather(_f64(I.rgb).to(device)))
    valid = lay.valid
    # alpha (neus_alpha)
    tc = _tr_dot3(dv, g)
    a = tr_clamp(0.5 + tr_scale(-tc, 0.5), lo=0.0)
    b = tr_clamp(-tc, lo=0.0)
    one_r = Tr(torch.tensor(1.0 - r32, dtype=F64), torch.tensor(abs(1.0 - r32), dtype=F64))
    ic = -(a * one_r + b * r32)
    icdt = tr_scale(ic * dt, 0.5)
    nxt, prv = sdf + icdt, sdf - icdt
    pc, nc = tr_sigmoid_fast(prv * s), tr_sigmoid_fast(nxt * s)
    q = ((pc - nc) + 1e-5) / (pc + 1e-5)
    alpha = tr_clamp(q, 0.0, 1.0)
    # colour head
    use_cal = I.head and I.img_idx is not None and I.weight_delta is not None
    if I.head:
        if use_cal:
            img = I.img_idx.detach().to(device).long().reshape(-1)
            cal = (img != int(I.fixed_img))
            wd = _f64(I.weight_delta).to(device)[img]
            bi = _f64(I.bias if I.bias is not None else torch.zeros_like(I.weight_delta)).to(device)[img]
            hw = Tr(torch.where(cal[:, None], 1.0 + wd, torch.ones_like(wd)), torch.where(cal[:, None], (1.0 + wd).abs(), torch.zeros_like(wd)))
            hb = Tr(torch.where(cal[:, None], bi, torch.zeros_like(bi)))
            hw = Tr(hw.v[:, None, :].expand(-1, lay.L, -1), hw.d[:, None, :].expand(-1, lay.L, -1))
            hb = Tr(hb.v[:, None, :].expand(-1, lay.L, -1))
            c = tr_sigmoid_exact(x * hw + hb)
        else:
            hw = Tr(torch.ones_like(x.v))
            c = tr_sigmoid_exact(x * 1.0 + 0.0)
    else:
        c = x
    res = {}
    if fwd_saved is None:
        al = alpha.where(valid, 0.0)
        # T_{i+1} = T_i (1 - alpha_i + 1e-7), left to right
        fac = (1.0 - al) + 1e-7
        rel = torch.where(valid & ~lay.last, fac.d / fac.v.abs() + 1.0, torch.zeros_like(fac.v))
        T_v = ClampedCumprod.apply(fac.v, valid, lay.last)[0]
        steps = torch.cumsum((valid & ~lay.last).to(F64), 1)
        T = Tr(T_v, T_v * (torch.cumsum(rel, 1) - rel) + TINY * steps)
        bgT = Tr(torch.cumprod(torch.where(valid & ~lay.last, fac.v, torch.ones_like(fac.v)), 1)[:, -1], None)
        bgT.d = bgT.v * rel.sum(1) + TINY * steps[:, -1]
        w = al * T
        wc = Tr(w.v[..., None] * c.v, w.d[..., None] * c.v.abs() + w.v.abs()[..., None] * c.d + TINY)    # fmaf: one rounding, in the sum
        pred = Tr(wc.v.sum(1), wc.d.sum(1) + torch.cumsum(wc.v, 1).abs().sum(1))
        wsum = tr_serial_sum(w, 1)
        ng = Tr(w.v[..., None] * g.v, w.d[..., None] * g.v.abs() + TINY)
        nws = Tr(ng.v.sum(1), ng.d.sum(1) + torch.cumsum(ng.v, 1).abs().sum(1))
        if I.bg_rgb is not None:
            bg = tr_exact(_f64(I.bg_rgb).to(device))
            tb = Tr(bgT.v[:, None] * bg.v, bgT.d[:, None] * bg.v.abs() + TINY)
            res["A_pred_bg"] = (tb.d + tb.v.abs())
            pred = Tr(pred.v + tb.v, pred.d + tb.d + (pred.v + tb.v).abs())
        comps, _, _ = _tr_normalize3(nws)
        res["A_normals"] = torch.stack([cc.d for cc in comps], 1)
        res["A_alpha"], rows = lay.scatter(alpha.d, N)
        res["A_T"], _ = lay.scatter(T.d, N)
        res["A_w"], _ = lay.scatter(w.d, N)
        res["A_pred"], res["A_wsum"], res["A_bgT"] = pred.d, wsum.d, bgT.d
        gt = tr_exact(_f64(I.gt_rgb).to(device)) if I.gt_rgb is not None else Tr(torch.zeros_like(pred.v))
        dlt = gt - pred
        l1 = (Tr(dlt.v[:, 0].abs(), dlt.d[:, 0]) + Tr(dlt.v[:, 1].abs(), dlt.d[:, 1])) + Tr(dlt.v[:, 2].abs(), dlt.d[:, 2])
        A_rl = [l1.d, torch.zeros_like(l1.d), torch.zeros_like(l1.d)]
        if I.gt_mask is not None:
            m = tr_exact(_f64(I.gt_mask).to(device).reshape(-1))
            p = tr_clamp(wsum, P_LO, P_HI)
            lp = tr_fn(p, torch.log, lambda v: 1.0 / v, 2.0)
            lq = tr_fn(1.0 - p, torch.log, lambda v: 1.0 / v, 2.0)
            bce = m * lp + (1.0 - m) * lq
            A_rl[1] = bce.d
        nrm = tr_sqrt(_tr_dot3(g, g)) - 1.0
        e = (nrm * nrm).where(valid, 0.0)
        depth = (lay.chunks + 5).to(F64).to(device)
        A_rl[2] = e.d.sum(1) + e.v.abs().sum(1) * depth
        res["A_ray_loss"] = torch.stack(A_rl, 1)
        res["rows"] = rows
        return res
    # ---------------------------------------------------------------- backward (at the saved forward values)
    al = tr_exact(lay.gather(fwd_saved["alpha"].detach().to(device).to(F64).reshape(-1)))
    fac = (1.0 - al) + 1e-7
    rel = torch.where(valid & ~lay.last, fac.d / fac.v.abs().clamp(min=1e-300) + 1.0, torch.zeros_like(fac.v))
    T_v = ClampedCumprod.apply(fac.v, valid, lay.last)[0]
    Ti = Tr(T_v, T_v * (torch.cumsum(rel, 1) - rel) + TINY * torch.cumsum((valid & ~lay.last).to(F64), 1))
    h = torch.ones(I.R, dtype=F64, device=device) if I.hit is None else (I.hit.detach().to(device).reshape(-1) != 0).to(F64)
    pred_s = fwd_saved["pred"].detach().to(device).to(F64).reshape(-1, 3)
    gt = _f64(I.gt_rgb).to(device)
    sg = torch.sign(pred_s - gt)
    gp_v = gtot * scale_rgb * h[:, None] * sg
    gp = Tr(gp_v, 2.0 * gp_v.abs())
    gws = Tr(torch.zeros(I.R, dtype=F64, device=device))
    if I.gt_mask is not None:
        ws = tr_exact(fwd_saved["wsum"].detach().to(device).to(F64).reshape(-1))
        m = tr_exact(_f64(I.gt_mask).to(device).reshape(-1))
        inside = (ws.v >= P_LO) & (ws.v <= P_HI)
        gm = Tr(torch.tensor(gtot * scale_mask, dtype=F64), torch.tensor(abs(gtot * scale_mask), dtype=F64))
        core = (-(m / ws.where(inside, 0.5))) + (1.0 - m) / (1.0 - ws.where(inside, 0.5))
        gws = (gm * core).where(inside, 0.0)
    ge = Tr(torch.tensor(gtot * scale_eik, dtype=F64), torch.tensor(2.0 * abs(gtot * scale_eik), dtype=F64))
    gbg = Tr(torch.zeros(I.R, dtype=F64, device=device))
    if I.bg_rgb is not None:
        bg = tr_exact(_f64(I.bg_rgb).to(device))
        bt = tr_exact(fwd_saved["bgT"].detach().to(device).to(F64).reshape(-1))
        gbg = _tr_dot3(gp, bg) * bt
        gb = Tr(gp.v * bt.v[:, None], gp.d * bt.v.abs()[:, None] + (gp.v * bt.v[:, None]).abs() + TINY)
        res["A_bg_rgb"] = gb.d
    gpL = Tr(gp.v[:, None, :].expand(-1, lay.L, -1), gp.d[:, None, :].expand(-1, lay.L, -1))
    gw = _tr_dot3(gpL, c) + Tr(gws.v[:, None].expand(-1, lay.L), gws.d[:, None].expand(-1, lay.L))
    gwww = (gw * al * Ti).where(valid, 0.0)
    S = tr_suffix(gwww)
    bcl = tr_clamp(fac, lo=1e-6)
    gbgL = Tr(gbg.v[:, None].expand(-1, lay.L), gbg.d[:, None].expand(-1, lay.L))
    ga = gw * Ti - ((S + gbgL) / bcl).where(valid & ~lay.last, 0.0)
    ga = Tr(ga.v, ga.d)
    den = pc + 1e-5
    dq_dpc = nc / (den * den)
    dq_dnc = -(1.0 / den)
    gpc = ((ga * dq_dpc) * pc) * (1.0 - pc)
    gnc = ((ga * dq_dnc) * nc) * (1.0 - nc)
    gsdf = (gpc + gnc) * s
    icd_v = torch.where(tc.v < 1.0, 0.5 * (1.0 - r32), 0.0) + torch.where(tc.v < 0.0, r32, 0.0)
    icd = Tr(torch.as_tensor(icd_v, dtype=F64), 2.0 * torch.as_tensor(icd_v, dtype=F64).abs())
    gic = tr_scale(((gnc - gpc) * s) * dt, 0.5)
    gtc = gic * icd
    gsa = (gpc * prv + gnc * nxt).where(valid, 0.0)
    nrm = tr_sqrt(_tr_dot3(g, g))
    ok = nrm.v > 0
    ek = ((ge * 2.0) * (nrm - 1.0) / nrm.where(ok, 1.0)).where(ok, 0.0)
    ogs = [gtc * _col(dv, k) + ek * _col(g, k) for k in range(3)]
    if I.gs is not None:
        gsv = tr_exact(lay.gather(_f64(I.gs).to(device)))
        A_, ia, oka = _tr_normalize3(g)
        B_, ib, okb = _tr_normalize3(gsv)
        dd = (A_[0] * B_[0] + A_[1] * B_[1]) + A_[2] * B_[2]
        inside = (dd.v >= -1.0 + 1e-6) & (dd.v <= 1.0 - 1e-6)
        one_m = 1.0 - dd * dd.where(inside, 0.0)
        ck = Tr(torch.tensor(curv_k, dtype=F64), torch.tensor(3.0 * abs(curv_k), dtype=F64))
        kk = -(ck * INV_PI) / tr_sqrt(one_m.where(inside, 1.0))
        o = []
        for k in range(3):
            ta = B_[k] - A_[k] * dd
            ta = Tr(torch.where(oka, ta.v, B_[k].v), torch.where(oka, ta.d, B_[k].d))
            ogs[k] = ogs[k] + ((kk * ta) * ia).where(inside, 0.0)
            tb = (A_[k] - B_[k] * dd)
            tb = Tr(torch.where(okb, tb.v, A_[k].v), torch.where(okb, tb.d, A_[k].d))
            o.append(((kk * tb) * ib).where(inside, 0.0))
        res["A_gs"], _ = lay.scatter(torch.stack([t.d for t in o], -1), N)
    wi = al * Ti
    qs = [_col(gpL, k) * wi for k in range(3)]
    if I.head:
        cc = [_col(c, k) for k in range(3)]
        v = [(qs[k] * cc[k]) * (1.0 - cc[k]) for k in range(3)]
        qs = [v[k] * _col(hw, k) for k in range(3)]
        if use_cal:
            xs = [_col(x, k) for k in range(3)]
            lane = torch.arange(lay.L, device=device) % 32
            img = I.img_idx.detach().to(device).long().reshape(-1)
            n_img = I.weight_delta.shape[0]
            A_w, A_b = torch.zeros(n_img, 3, dtype=F64, device=device), torch.zeros(n_img, 3, dtype=F64, device=device)
            cal = (img != int(I.fixed_img)) & ~lay.skip.to(device)
            # per ray: each lane sums its chunk terms serially, then a 5-level tree; the rays of an image meet in float atomics
            cnt = torch.zeros(n_img, dtype=F64, device=device).index_add_(0, img[cal], torch.ones(int(cal.sum()), dtype=F64, device=device))
            for k in range(3):
                for tgt, term in ((A_w, (v[k] * xs[k]).where(valid, 0.0)), (A_b, v[k].where(valid, 0.0))):
                    depth = (lay.chunks + 5).to(F64).to(device)
                    per_ray = term.d.sum(1) + term.v.abs().sum(1) * depth
                    tot = term.v.sum(1).abs()
                    a_ray = per_ray + tot * cnt[img]
                    tgt[:, k].index_add_(0, img[cal], a_ray[cal])
            res["A_wd"], res["A_bias"] = A_w, A_b
    res["A_sdf"], rows = lay.scatter(gsdf.d, N)
    res["A_grad"], _ = lay.scatter(torch.stack([t.d for t in ogs], -1), N)
    res["A_rgb"], _ = lay.scatter(torch.stack([t.d for t in qs], -1), N)
    depth = (lay.chunks + 5).to(F64).to(device)
    n_act = float((~lay.skip).sum())
    res["A_inv_s"] = (gsa.d.sum() + (gsa.v.abs().sum(1) * depth).sum() + gsa.v.sum(1).abs().sum() * n_act).reshape(1)
    res["rows"] = rows
    return res


# ------------------------------------------------------------------------------------------------ psdf_loss_terms
def softplus(x):
    return F.softplus(x, beta=1.0, threshold=20.0)


def loss_terms_reference(N, nv, n_mean, grad, gs, R, ray_loss, sdf_off, c_rgb, c_mask, w_eik, w_curv, w_curv_dev, w_off, w_lip, lip_c,
                         leaves=False):
    """fp64 psdf_loss_terms. Returns dict(loss, terms [10], g_off [n_off], and the error scales A_loss, A_terms, A_g_off)."""
    rl = ray_loss.detach().double().cpu().reshape(R, 3)
    cnt = max(int(n_mean) if n_mean is not None else nv, 1)
    nb = max(-(-max(N if gs is not None else 0, R, 1 if sdf_off is None else sdf_off.numel(), 1) // 256), 1)
    depth = 5 + 8 + nb + 1             # warp tree, block sum, atomics across blocks, the final read
    l1, bce, eik = rl[:, 0].sum(), rl[:, 1].sum(), rl[:, 2].sum()
    A = {k: rl[:, i].abs().sum() * depth for i, k in enumerate(("l1", "bce", "eik"))}
    curv_mean, A_curv = torch.tensor(0.0, dtype=F64), torch.tensor(0.0, dtype=F64)
    if gs is not None:
        g = grad.detach().double().cpu()[:nv]
        s = gs.detach().double().cpu()[:nv]
        dot = (F.normalize(g, dim=1, eps=1e-12) * F.normalize(s, dim=1, eps=1e-12)).sum(1)
        dc = dot.clamp(-1.0 + 1e-6, 1.0 - 1e-6)
        curv = torch.acos(dc) / math.pi
        inside = dc == dot
        # the dot of two normalised vectors: 3 normalisations (~4 u each) and 5 roundings, through acos' = 1 / sqrt(1 - d^2)
        A_dot = 14.0 * (g.abs() / g.norm(dim=1, keepdim=True).clamp(min=1e-12) * (s.abs() / s.norm(dim=1, keepdim=True).clamp(min=1e-12))).sum(1)
        A_c = torch.where(inside, A_dot / torch.sqrt(1.0 - dc * dc), torch.zeros_like(dc)) / math.pi + 6.0 * curv
        curv_mean = curv.sum() / cnt
        A_curv = (A_c.sum() + curv.sum() * depth) / cnt + curv_mean.abs()
    off_mean, A_off, g_off, A_goff = torch.tensor(0.0, dtype=F64), torch.tensor(0.0, dtype=F64), None, None
    if sdf_off is not None:
        so = sdf_off.detach().double().cpu().reshape(-1)
        e = torch.exp(-100.0 * so.abs())
        n_off = so.numel()
        off_mean = e.sum() / n_off
        # expf 2 ulp of a value whose argument carries 1 rounding (100 |s|): 4 + |100 s| u relative
        A_e = e * (4.0 + 100.0 * so.abs())
        A_off = (A_e.sum() + e.sum() * depth) / n_off + off_mean
        g_off = w_off / n_off * (-100.0 * torch.sign(so)) * e
        A_goff = g_off.abs() * 4.0 + (w_off / n_off * 100.0 * torch.sign(so).abs()) * A_e
    lip, A_lip = torch.tensor(0.0, dtype=F64), torch.tensor(0.0, dtype=F64)
    if w_lip != 0.0:
        lip = torch.tensor(1.0, dtype=F64)
        for c in lip_c:
            lip = lip * softplus(c.detach().double().cpu().reshape(()))
        A_lip = lip * 4 * 4.0
    wc = w_curv * (float(w_curv_dev) if w_curv_dev is not None else 1.0)
    loss = l1 * c_rgb + bce * c_mask + eik * (w_eik / cnt)
    A_loss = (A["l1"] + l1.abs()) * abs(c_rgb) + (A["bce"] + bce.abs()) * abs(c_mask) + (A["eik"] + 2 * eik.abs()) * abs(w_eik / cnt)
    if gs is not None:
        loss = loss + curv_mean * wc
        A_loss = A_loss + (A_curv + 2 * curv_mean.abs()) * abs(wc)
    if sdf_off is not None:
        loss = loss + off_mean * w_off
        A_loss = A_loss + (A_off + off_mean.abs()) * abs(w_off)
    if w_lip != 0.0:
        loss = loss + lip * w_lip
        A_loss = A_loss + (A_lip + lip.abs()) * abs(w_lip)
    A_loss = A_loss + 6.0 * abs(float(loss))
    terms = torch.stack([l1, bce, eik, curv_mean, off_mean, lip, torch.tensor(float(nv), dtype=F64), torch.tensor(float(cnt), dtype=F64),
                         l1 * c_rgb, eik / cnt])
    A_terms = torch.stack([A["l1"], A["bce"], A["eik"], A_curv, A_off, A_lip, torch.tensor(0.0, dtype=F64), torch.tensor(0.0, dtype=F64),
                           (A["l1"] + l1.abs()) * abs(c_rgb), (A["eik"] + eik.abs()) / cnt])
    return dict(loss=loss.reshape(1), terms=terms, g_off=g_off, A_loss=A_loss.reshape(1), A_terms=A_terms, A_g_off=A_goff)
