"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

fp64 reference of the fused kernels: the three training backwards (csrc/fused_sdf_bwd.cu, fused_rgb_bwd.cu, fused_bg.cu) and the
forwards (fused_sdf.cu: value + tangent, value-only and sphere-tracer kernels; fused_rgb.cu; fused_bg.cu). The same operations as the
kernels, with every reduction in fp64, so that a kernel can be judged per level, per layer and per element rather than by one ratio
per tensor.

"The same operation" is defined as follows. The discrete decisions of the permutohedral encoder (remainder-0 point, rank, hashed
vertex indices) and the barycentric weights are taken in fp32 from encoding_oracle, which the per-op encoder matches bit for bit. At
the fine levels (pos + shift) * scale reaches ~7e4, where fp32 moves the barycentric weights by ~1e-2; the kernels share that, so it
is not an error of theirs. Everything downstream is fp64: feature sums, the MLPs (exact-erf GELU), softplus, the normal
normalisation, the reverse sweep, weight / bias gradients and the lattice scatter. The derivative of a barycentric weight with
respect to the position is the exact fp64 one (constant inside a simplex); in the autograd formulation it enters through a
straight-through term whose value is the fp32 weight. Spherical-harmonics inputs come from the fp32 C oracle, as in the kernels.

Two formulations are provided. `*_reference` runs the MLPs with an explicit tangent stream (the SDF's <g_grad, grad sdf> term is the
directional derivative along g_grad) under fp64 autograd and returns the per-sample encoder gradients abar_0 (and tabar_0), from
which the lattice gradient is formed by an explicit fp64 index_add together with, per table entry, A = sum |contribution| and
n = the number of (sample, vertex) contributions. `*_autograd` differentiates the whole forward (double backward for the SDF) with
the lattice as an autograd leaf; tests/test_backward_fp64_reference_cpu.py checks that the two agree to 1e-12.

The forward references (`*_forward_reference`) return, beside every output, its error scale A: the linearised propagation of the
terms that form it, i.e. what the output's rounding error is proportional to when every operand of every product carries a small
relative error. A kernel output is accepted per element when |got - ref| <= eps A (tests/test_forward_fp64_reference_cpu.py derives
eps and shows that the kernels' arithmetic, emulated, stays well inside it while a one-pass bf16 product does not):
  * layer-0 input A^a_0: w_l sum_k |B_k| |v_k| for the two columns of level l, |x * scaling| for the concat columns; colour inputs add
    |SH|, |normal| and |geom|, background inputs |SH|. An input's error is its own bf16 split, relative to its value, so its scale is
    the absolute sum (>= |value|);
  * every layer: A^z_l = sqrt(W_l^2 (A^a_l)^2 + b_l^2), then A^a_{l+1} = sqrt((gelu'(z_l) A^z_l)^2 + a_{l+1}^2). The rounding errors of a
    product's K terms are independent, so they add in quadrature: the absolute sum |W_l| A^a_l + |b_l| overstates them by ~sqrt(K)
    per layer, compounding with depth (2^9 over the background's seven layers of 64), so that no single eps would both accept the
    kernels' hidden-16 SDF and reject a one-pass product in the background network. The first term of A^a carries an error of z_l
    through the activation; the second is the activation's own representation error (the next product splits a_{l+1} itself): near
    z = -0.75 (gelu' = 0) the first vanishes while |gelu(z)| = 0.17 |z| does not;
  * the density: |sigmoid(z)| A^z (softplus' = sigmoid);
  * tangent streams (d / dx_j, input A^{ta}_0 = w_l sum_k |dB_k| |v_k| and the concat column's |scaling|): A^{tz}_l = sqrt(W_l^2
    (A^{ta}_l)^2), A^{ta}_{l+1} = sqrt((gelu'(z_l) A^{tz}_l)^2 + (gelu''(z_l) tz_l A^z_l)^2 + ta_{l+1}^2); the middle term is where an
    error of z_l enters the gradient through the GELU, the last the tangent's own representation error.
"""
import math

import numpy as np
import torch

from . import encoding_oracle as eo

F64 = torch.float64


def level_scales(L, D):
    """scale factors of models.make_encoding: geomspace(1, 1e-4, L) sigmas -> [L, D] fp32"""
    return eo.scale_factor([float(s) for s in np.geomspace(1.0, 0.0001, num=L)], D)


def window_of(L, t):
    """the coarse-to-fine window at ramp position t (Coarse2Fine), fp32 [L]"""
    return eo.coarse2fine(L, t).float()


# ------------------------------------------------------------------------------------------------ encoder
class Plan:
    """discrete decisions and fp32 barycentric weights of every level, from encoding_oracle on the CPU"""

    def __init__(self, pos, scale, shift, T):
        pos = pos.detach().cpu().float()
        self.N, self.D = pos.shape
        self.L, self.T = scale.shape[0], int(T)
        self.rank, self.rem0, self.idx, self.bary = [], [], [], []
        with torch.no_grad():
            for l in range(self.L):
                sh = shift[l].cpu().float() if shift is not None else torch.zeros(self.D)
                rem0, rank, bary = eo.simplex(pos, scale[l].cpu().float(), sh)
                self.rem0.append(rem0)
                self.rank.append(rank)
                self.idx.append(eo.vertex_indices(rem0, rank, self.T))
                self.bary.append(bary.double())
        self.scale = scale.detach().cpu().double()
        self.shift = shift.detach().cpu().double() if shift is not None else torch.zeros(self.L, self.D, dtype=F64)

    def to(self, device):
        for k in ("rank", "rem0", "idx", "bary"):
            setattr(self, k, [t.to(device) for t in getattr(self, k)])
        self.scale, self.shift = self.scale.to(device), self.shift.to(device)
        return self


def bary_linear(cf, rank, rem0=None):
    """the barycentric weights as the affine function of the scaled coordinates cf [N, D] they are inside the simplex of (rank,
    rem0), in cf's dtype. rem0 = None: the linear part only, i.e. the tangent of the weights along a direction whose scaled
    coordinates are cf."""
    N, D = cf.shape
    sm = torch.zeros(N, dtype=cf.dtype, device=cf.device)
    E = [None] * (D + 1)
    for i in range(D, 0, -1):
        E[i] = sm - i * cf[:, i - 1]
        sm = sm + cf[:, i - 1]
    E[0] = sm
    E = torch.stack(E, 1)
    if rem0 is not None:
        E = E - rem0.to(cf.dtype)
    delta = E / (D + 1)
    b = torch.zeros(N, D + 2, dtype=cf.dtype, device=cf.device)
    b = b.scatter_add(1, D - rank, delta).scatter_add(1, D + 1 - rank, -delta)
    b0 = b[:, 0] + b[:, D + 1] + (1.0 if rem0 is not None else 0.0)
    return torch.cat([b0[:, None], b[:, 1:D + 1]], 1)


def _gather(lattice64, plan, l):
    return lattice64[l][plan.idx[l]]                         # [N, D+1, F]


def encode_st(pos64, lattice64, plan, window, points_scaling):
    """differentiable encoding (fp64): value = fp32 barycentric weights, position derivative = the exact fp64 one (straight-through)"""
    cols = []
    w = window.double().to(pos64.device)
    for l in range(plan.L):
        cf = (pos64 + plan.shift[l]) * plan.scale[l]
        lin = bary_linear(cf, plan.rank[l], plan.rem0[l])
        B = plan.bary[l] + (lin - lin.detach())
        cols.append(w[l] * (B[:, :, None] * _gather(lattice64, plan, l)).sum(1))
    return torch.cat(cols + _concat(pos64, points_scaling), 1)


def _concat(x64, points_scaling):
    """concat-point columns: x * scaling, zero-padded to an even count (F = 2)"""
    N, D = x64.shape
    cols = [x64 * points_scaling]
    if D % 2:
        cols.append(torch.zeros(N, 1, dtype=F64, device=x64.device))
    return cols


def features(plan, lattice64, pos64, window, points_scaling, v64=None):
    """encoder values (and, with v64, their tangent along v) as plain fp64 tensors -> feat [N, 2L + E], tfeat or None, per level
    (B, dB) with dB = the tangent of the barycentric weights"""
    w = window.double().to(pos64.device)
    cols, tcols, per_level = [], [], []
    for l in range(plan.L):
        vals = _gather(lattice64, plan, l)
        B = plan.bary[l]
        cols.append(w[l] * (B[:, :, None] * vals).sum(1))
        dB = None
        if v64 is not None:
            dB = bary_linear(v64 * plan.scale[l], plan.rank[l])
            tcols.append(w[l] * (dB[:, :, None] * vals).sum(1))
        per_level.append((B, dB))
    feat = torch.cat(cols + _concat(pos64, points_scaling), 1)
    tfeat = torch.cat(tcols + _concat(v64, points_scaling), 1) if v64 is not None else None
    return feat, tfeat, per_level


def lattice_scatter(plan, window, per_level, abar0, tabar0=None, abar_abs=None, tabar_abs=None):
    """explicit fp64 lattice gradient from the per-sample encoder gradients: per level (grad [T, 2], A = sum |contribution| [T, 2],
    n = contributions per entry [T], A_terms [T, 2]). A_terms is A with abar_0 (tabar_0) replaced by the sum of the absolute terms of the
    product that forms it, |zbar_1| |W_0| (abar_abs, tabar_abs): the scale of a GEMM output's rounding error where its terms cancel."""
    w = window.double().to(abar0.device)
    out = []
    for l in range(plan.L):
        B, dB = per_level[l]
        a = abar0[:, 2 * l:2 * l + 2]
        c = w[l] * B[:, :, None] * a[:, None, :]                              # [N, D+1, 2]
        if tabar0 is not None:
            c = c + w[l] * dB[:, :, None] * tabar0[:, None, 2 * l:2 * l + 2]
        idx = plan.idx[l].reshape(-1)
        c = c.reshape(-1, 2)
        g = torch.zeros(plan.T, 2, dtype=F64, device=c.device).index_add_(0, idx, c)
        A = torch.zeros(plan.T, 2, dtype=F64, device=c.device).index_add_(0, idx, c.abs())
        n = torch.zeros(plan.T, dtype=F64, device=c.device).index_add_(0, idx, torch.ones_like(c[:, 0]))
        At = A
        if abar_abs is not None:
            t = w[l] * B.abs()[:, :, None] * abar_abs[:, None, 2 * l:2 * l + 2]
            if tabar_abs is not None:
                t = t + w[l] * dB.abs()[:, :, None] * tabar_abs[:, None, 2 * l:2 * l + 2]
            At = torch.zeros(plan.T, 2, dtype=F64, device=c.device).index_add_(0, idx, t.reshape(-1, 2))
        out.append((g, A, n, At))
    return out


# ------------------------------------------------------------------------------------------------ MLP pieces
SQRT1_2 = 1.0 / math.sqrt(2.0)
INV_SQRT_2PI = 1.0 / math.sqrt(2.0 * math.pi)


def gelu(z):
    return z * 0.5 * (1.0 + torch.erf(z * SQRT1_2))


def gelu_d1(z):
    return 0.5 * (1.0 + torch.erf(z * SQRT1_2)) + z * torch.exp(-0.5 * z * z) * INV_SQRT_2PI


class Layers:
    """linear layers whose inputs / pre-activations (and tangents) are kept so that A = |zbar|^T |a| can be formed afterwards"""

    def __init__(self, W, b, device):
        self.W = [w.detach().to(device).double().requires_grad_(True) for w in W]
        self.b = [x.detach().to(device).double().requires_grad_(True) for x in b]
        self.a, self.z, self.ta, self.tz = [], [], [], []

    def __call__(self, l, a, ta=None):
        z = a @ self.W[l].t() + self.b[l]
        self.a.append(a)
        self.z.append(z)
        tz = None
        if ta is not None:
            tz = ta @ self.W[l].t()
            self.ta.append(ta)
            self.tz.append(tz)
        return z, tz

    def grads(self, loss, extra):
        """-> gradients of `extra`, of W, of b; and A_W, A_b per layer"""
        nl = len(self.W)
        wrt = list(extra) + self.W + self.b + self.z + self.tz
        g = torch.autograd.grad(loss, wrt, allow_unused=True)
        g = [torch.zeros_like(t) if x is None else x for x, t in zip(g, wrt)]
        ne = len(extra)
        ge, gW, gb = g[:ne], g[ne:ne + nl], g[ne + nl:ne + 2 * nl]
        zb, tzb = g[ne + 2 * nl:ne + 3 * nl], g[ne + 3 * nl:]
        AW, Ab = [], []
        for l in range(nl):
            A = zb[l].abs().t() @ self.a[l].detach().abs()
            if self.tz:
                A = A + tzb[l].abs().t() @ self.ta[l].detach().abs()
            AW.append(A)
            Ab.append(zb[l].abs().sum(0))
        self.zbar, self.tzbar = [z.detach() for z in zb], [z.detach() for z in tzb]
        return ge, [x.detach() for x in gW], [x.detach() for x in gb], AW, Ab, self.zbar


def _dev(device):
    return torch.device(device) if device is not None else torch.device("cpu")


def _result(lat, gW, gb, AW, Ab, **kw):
    r = dict(lattice=lat, W=gW, b=gb, A_W=AW, A_b=Ab)
    r.update(kw)
    return r


# ------------------------------------------------------------------------------------------------ SDF
def sdf_reference(pos, lattice, scale, shift, window, points_scaling, W, b, g_sdf, g_grad, g_geom, device=None, plan=None):
    """gradients of  sum g_sdf sdf + sum g_geom geom + sum <g_grad, d sdf / dx>  (any upstream may be None) wrt the lattice, W_l, b_l.
    -> dict: lattice = per level (grad, A, n), W, b, A_W, A_b, abar0, tabar0, sdf, geom"""
    dev = _dev(device)
    N = pos.shape[0]
    plan = plan or Plan(pos, scale, shift, lattice.shape[1]).to(dev)
    lat = lattice.detach().to(dev).double()
    pos64 = pos.detach().to(dev).double()
    v64 = g_grad.detach().to(dev).double() if g_grad is not None else torch.zeros_like(pos64)
    feat, tfeat, per_level = features(plan, lat, pos64, window, points_scaling, v64)
    feat.requires_grad_(True)
    tfeat.requires_grad_(True)
    net = Layers(W, b, dev)
    a, ta = feat, tfeat
    for l in range(4):
        z, tz = net(l, a, ta)
        if l < 3:
            d1 = gelu_d1(z)
            a, ta = gelu(z), d1 * tz
    loss = (z[:, 0] * 0).sum()
    if g_sdf is not None:
        loss = loss + (z[:, 0] * g_sdf.detach().to(dev).double().reshape(-1)).sum()
    if g_geom is not None and z.shape[1] > 1:
        loss = loss + (z[:, 1:] * g_geom.detach().to(dev).double().reshape(N, -1)).sum()
    if g_grad is not None:
        loss = loss + tz[:, 0].sum()
    (abar0, tabar0), gW, gb, AW, Ab, _ = net.grads(loss, [feat, tfeat])
    W0a = net.W[0].detach().abs()
    lat_out = lattice_scatter(plan, window, per_level, abar0, tabar0, net.zbar[0].abs() @ W0a, net.tzbar[0].abs() @ W0a)
    return _result(lat_out, gW, gb, AW, Ab, abar0=abar0, tabar0=tabar0, sdf=z[:, :1].detach(), geom=z[:, 1:].detach(), plan=plan)


def sdf_autograd(pos, lattice, scale, shift, window, points_scaling, W, b, g_sdf, g_grad, g_geom):
    """the same gradients by fp64 autograd through the whole forward: d sdf / dx by a first backward (create_graph), then the loss'
    backward with the lattice as a leaf. -> (lattice grad [L, T, 2], [gW], [gb], loss)"""
    plan = Plan(pos, scale, shift, lattice.shape[1])
    lat = lattice.detach().double().requires_grad_(True)
    p = pos.detach().double().requires_grad_(True)
    Ws = [w.detach().double().requires_grad_(True) for w in W]
    bs = [x.detach().double().requires_grad_(True) for x in b]
    h = encode_st(p, lat, plan, window, points_scaling)
    for l in range(4):
        h = torch.nn.functional.linear(h, Ws[l], bs[l])
        if l < 3:
            h = torch.nn.functional.gelu(h)
    sdf = h[:, 0]
    gx = torch.autograd.grad(sdf.sum(), p, create_graph=True)[0]
    loss = (sdf * 0).sum()
    if g_sdf is not None:
        loss = loss + (sdf * g_sdf.double().reshape(-1)).sum()
    if g_geom is not None and h.shape[1] > 1:
        loss = loss + (h[:, 1:] * g_geom.double()).sum()
    if g_grad is not None:
        loss = loss + (gx * g_grad.double()).sum()
    g = torch.autograd.grad(loss, [lat] + Ws + bs, allow_unused=True)
    z = lambda t, ref: torch.zeros_like(ref) if t is None else t.detach()
    return z(g[0], lat), [z(x, w) for x, w in zip(g[1:5], Ws)], [z(x, w) for x, w in zip(g[5:], bs)], loss.detach()


# ------------------------------------------------------------------------------------------------ colour network
def _normalize64(g):
    return g / g.norm(dim=1, keepdim=True).clamp(min=1e-12)                 # F.normalize(eps = 1e-12)


def sh_fp32(dirs, degree):
    """real spherical harmonics from the fp32 C oracle, as fp64"""
    from . import rayops as ro
    return torch.from_numpy(ro.spherical_harmonics(dirs.detach().cpu().float().numpy(), degree)).double()


def rgb_reference(pos, dirs, sdf_grad, geom, lattice, scale, shift, window, points_scaling, W_eff, b, g_out, device=None, sh=None):
    """gradients of  sum g_out out  for out = MLP([enc(pos) | SH_5(dirs) | normalize(sdf_grad) | geom]) (W_eff: the normalised matrices
    the kernels receive) wrt the lattice, W_eff, b, sdf_grad and geom. -> dict: lattice, W, b, A_W, A_b, g_sdf_grad, A_sdf_grad, g_geom,
    A_geom, abar0, out"""
    dev = _dev(device)
    plan = Plan(pos, scale, shift, lattice.shape[1]).to(dev)
    lat = lattice.detach().to(dev).double()
    pos64 = pos.detach().to(dev).double()
    feat, _, per_level = features(plan, lat, pos64, window, points_scaling)
    sh = (sh if sh is not None else sh_fp32(dirs, 5)).to(dev)
    sg = sdf_grad.detach().to(dev).double().requires_grad_(True)
    gm = geom.detach().to(dev).double().requires_grad_(True)
    feat.requires_grad_(True)
    nrm = _normalize64(sg)
    x = torch.cat([feat, sh, nrm, gm], 1)
    net = Layers(W_eff, b, dev)
    a = x
    for l in range(4):
        z, _ = net(l, a)
        if l < 3:
            a = gelu(z)
    loss = (z * g_out.detach().to(dev).double()).sum()
    (abar0, g_sg, g_gm), gW, gb, AW, Ab, zb = net.grads(loss, [feat, sg, gm])
    # A of the per-sample outputs: |zbar_1| |W_0| over the input columns, then through |d normalize / d g| for the sdf gradient
    Ax = zb[0].abs() @ net.W[0].detach().abs()
    E = feat.shape[1]
    A_geom = Ax[:, E + 28:E + 60]
    gd = sg.detach()
    r = gd.norm(dim=1, keepdim=True).clamp(min=1e-12)
    n = gd / r
    J = (torch.eye(3, dtype=F64, device=dev)[None] - n[:, :, None] * n[:, None, :]) / r[:, :, None]
    A_sg = (J.abs() * Ax[:, E + 25:E + 28, None]).sum(1)
    lat_out = lattice_scatter(plan, window, per_level, abar0, None, Ax)
    return _result(lat_out, gW, gb, AW, Ab, g_sdf_grad=g_sg.detach(), A_sdf_grad=A_sg, g_geom=g_gm.detach(), A_geom=A_geom, abar0=abar0,
                   out=z.detach(), plan=plan)


def rgb_autograd(pos, dirs, sdf_grad, geom, lattice, scale, shift, window, points_scaling, W_eff, b, g_out):
    """the colour gradients by fp64 autograd with the lattice as a leaf -> (lattice grad, [gW], [gb], g_sdf_grad, g_geom)"""
    plan = Plan(pos, scale, shift, lattice.shape[1])
    lat = lattice.detach().double().requires_grad_(True)
    sg = sdf_grad.detach().double().requires_grad_(True)
    gm = geom.detach().double().requires_grad_(True)
    Ws = [w.detach().double().requires_grad_(True) for w in W_eff]
    bs = [x.detach().double().requires_grad_(True) for x in b]
    h = torch.cat([encode_st(pos.detach().double(), lat, plan, window, points_scaling), sh_fp32(dirs, 5), _normalize64(sg), gm], 1)
    for l in range(4):
        h = torch.nn.functional.linear(h, Ws[l], bs[l])
        if l < 3:
            h = torch.nn.functional.gelu(h)
    g = torch.autograd.grad((h * g_out.double()).sum(), [lat] + Ws + bs + [sg, gm])
    return g[0], list(g[1:5]), list(g[5:9]), g[9], g[10]


# ------------------------------------------------------------------------------------------------ background network
def bg_reference(pos, dirs, lattice, scale, shift, window, points_scaling, W, b, g_rgb, g_density, device=None, sh=None):
    """gradients of  sum g_rgb rgb_raw + sum g_density density  of the 7-layer NerfHash MLP on the 4-D encoding wrt the lattice, W_l,
    b_l (torch.nn.Linear layout, trunk layer 3 unrotated). -> dict: lattice, W, b, A_W, A_b, abar0, rgb, density"""
    dev = _dev(device)
    plan = Plan(pos, scale, shift, lattice.shape[1]).to(dev)
    lat = lattice.detach().to(dev).double()
    pos64 = pos.detach().to(dev).double()
    feat, _, per_level = features(plan, lat, pos64, window, points_scaling)
    feat.requires_grad_(True)
    sh = (sh if sh is not None else sh_fp32(dirs, 4)).to(dev)
    net = Layers(W, b, dev)
    a = feat
    for l in range(4):
        z, _ = net(l, a)
        if l < 3:
            a = gelu(z)
    density = torch.nn.functional.softplus(z[:, :1])
    a = torch.cat([gelu(z[:, 1:65]), sh], 1)
    for l in range(4, 7):
        z, _ = net(l, a)
        if l < 6:
            a = gelu(z)
    loss = (z * g_rgb.detach().to(dev).double()).sum() + (density * g_density.detach().to(dev).double().reshape(-1, 1)).sum()
    (abar0,), gW, gb, AW, Ab, _ = net.grads(loss, [feat])
    lat_out = lattice_scatter(plan, window, per_level, abar0, None, net.zbar[0].abs() @ net.W[0].detach().abs())
    return _result(lat_out, gW, gb, AW, Ab, abar0=abar0, rgb=z.detach(), density=density.detach(), plan=plan)


def bg_autograd(pos, dirs, lattice, scale, shift, window, points_scaling, W, b, g_rgb, g_density):
    """the background gradients by fp64 autograd with the lattice as a leaf -> (lattice grad, [gW], [gb])"""
    plan = Plan(pos, scale, shift, lattice.shape[1])
    lat = lattice.detach().double().requires_grad_(True)
    Ws = [w.detach().double().requires_grad_(True) for w in W]
    bs = [x.detach().double().requires_grad_(True) for x in b]
    h = encode_st(pos.detach().double(), lat, plan, window, points_scaling)
    for l in range(4):
        h = torch.nn.functional.linear(h, Ws[l], bs[l])
        if l < 3:
            h = torch.nn.functional.gelu(h)
    density = torch.nn.functional.softplus(h[:, :1])
    h = torch.cat([torch.nn.functional.gelu(h[:, 1:65]), sh_fp32(dirs, 4)], 1)
    for l in range(4, 7):
        h = torch.nn.functional.linear(h, Ws[l], bs[l])
        if l < 6:
            h = torch.nn.functional.gelu(h)
    loss = (h * g_rgb.double()).sum() + (density * g_density.double().reshape(-1, 1)).sum()
    g = torch.autograd.grad(loss, [lat] + Ws + bs)
    return g[0], list(g[1:8]), list(g[8:])


def dense_lattice(lat_out):
    """per-level (grad, A, n) -> [L, T, 2] gradient"""
    return torch.stack([o[0] for o in lat_out], 0)


# ------------------------------------------------------------------------------------------------ forwards with error scales
def gelu_d2(z):
    return torch.exp(-0.5 * z * z) * INV_SQRT_2PI * (2.0 - z * z)


class Exact:
    """the arithmetic of the forward references: fp64 products and the exact-erf GELU. A test may substitute an emulation of a
    kernel's arithmetic (same interface) to run the same chain as the kernel would."""

    def linear(self, l, a, W, b=None):
        z = a @ W.t()
        return z + b if b is not None else z

    def gelu(self, z):
        """-> gelu(z), gelu'(z)"""
        return gelu(z), gelu_d1(z)


def features_bound(plan, lattice64, pos64, window, points_scaling, tangents=False):
    """encoder values and their A (see the module docstring); with tangents, the three tangents d / dx_j and their A as [3, N, E]"""
    w = window.double().to(pos64.device)
    N, D = pos64.shape
    cols, acols, tcols, atcols = [], [], [], []
    dirs = torch.eye(D, dtype=F64, device=pos64.device) if tangents else None
    for l in range(plan.L):
        vals = _gather(lattice64, plan, l)
        B = plan.bary[l]
        cols.append(w[l] * (B[:, :, None] * vals).sum(1))
        acols.append(w[l] * (B.abs()[:, :, None] * vals.abs()).sum(1))
        if tangents:
            dB = torch.stack([bary_linear(dirs[j].expand(N, D) * plan.scale[l], plan.rank[l]) for j in range(D)], 0)    # [3, N, D+1]
            tcols.append(w[l] * (dB[..., None] * vals[None]).sum(2))
            atcols.append(w[l] * (dB.abs()[..., None] * vals.abs()[None]).sum(2))
    cc = _concat(pos64, points_scaling)
    feat = torch.cat(cols + cc, 1)
    A = torch.cat(acols + [c.abs() for c in cc], 1)
    if not tangents:
        return feat, A, None, None
    tc = torch.stack([torch.cat(_concat(dirs[j].expand(N, D), points_scaling), 1) for j in range(D)], 0)
    tfeat = torch.cat([torch.cat(tcols, 2), tc], 2)
    At = torch.cat([torch.cat(atcols, 2), tc.abs()], 2)
    return feat, A, tfeat, At


def chain_bound(ar, layers, a, A, ta=None, At=None, first=0):
    """Linear -> GELU -> ... -> Linear over layers [(W, b)] (fp64) with the error scales of the module docstring. Returns the last
    pre-activation z and A^z, and the tangents tz, A^{tz} (or None)."""
    n = len(layers)
    for i, (W, b) in enumerate(layers):
        W2 = W * W
        z = ar.linear(first + i, a, W, b)
        Az = (A * A @ W2.t() + b * b).sqrt()
        tz = Atz = None
        if ta is not None:
            tz = ar.linear(first + i, ta, W)
            Atz = (At * At @ W2.t()).sqrt()
        if i == n - 1:
            return z, Az, tz, Atz
        a, d1 = ar.gelu(z)
        A = ((d1 * Az) ** 2 + a.double() ** 2).sqrt()
        if ta is not None:
            z64 = z.double()
            ta = d1 * tz
            At = ((d1 * Atz) ** 2 + (gelu_d2(z64) * tz * Az) ** 2 + ta.double() ** 2).sqrt()


def _dev_layers(W, b, dev):
    return [(w.detach().to(dev).double(), x.detach().to(dev).double()) for w, x in zip(W, b)]


def sdf_forward_reference(pos, lattice, scale, shift, window, points_scaling, W, b, device=None, plan=None, arith=None):
    """the SDF forward: sdf [N], grad = d sdf / dx [N, 3] (three tangent streams), geom [N, out_dim - 1] and their error scales
    A_sdf, A_grad, A_geom (module docstring)"""
    dev = _dev(device)
    ar = arith or Exact()
    plan = plan or Plan(pos, scale, shift, lattice.shape[1]).to(dev)
    feat, A, tfeat, At = features_bound(plan, lattice.detach().to(dev).double(), pos.detach().to(dev).double(), window, points_scaling, True)
    z, Az, tz, Atz = chain_bound(ar, _dev_layers(W, b, dev), feat, A, tfeat, At)
    z, tz = z.double(), tz.double()
    return dict(sdf=z[:, 0], grad=tz[:, :, 0].t(), geom=z[:, 1:], A_sdf=Az[:, 0], A_grad=Atz[:, :, 0].t(), A_geom=Az[:, 1:], plan=plan)


def lipschitz_weights(W, c):
    """LipshitzMLP.normalization in fp64: W * min(softplus(c) / sum_k |W|, 1) per row"""
    W, c = W.double(), torch.as_tensor(c).double().reshape(())
    return W * torch.clamp(torch.nn.functional.softplus(c) / W.abs().sum(1), max=1.0)[:, None]


def rgb_forward_reference(pos, dirs, sdf_grad, geom, lattice, scale, shift, window, points_scaling, W_eff, b, device=None, sh=None,
                          arith=None):
    """the colour network's linear output out [N, 3] and A_out, W_eff the normalised matrices"""
    dev = _dev(device)
    ar = arith or Exact()
    plan = Plan(pos, scale, shift, lattice.shape[1]).to(dev)
    feat, A, _, _ = features_bound(plan, lattice.detach().to(dev).double(), pos.detach().to(dev).double(), window, points_scaling)
    sh = (sh if sh is not None else sh_fp32(dirs, 5)).to(dev)
    nrm = _normalize64(sdf_grad.detach().to(dev).double())
    gm = geom.detach().to(dev).double()
    x = torch.cat([feat, sh, nrm, gm], 1)
    Ax = torch.cat([A, sh.abs(), nrm.abs(), gm.abs()], 1)
    z, Az, _, _ = chain_bound(ar, _dev_layers(W_eff, b, dev), x, Ax)
    return dict(out=z.double(), A_out=Az)


def bg_forward_reference(pos, dirs, lattice, scale, shift, window, points_scaling, W, b, device=None, sh=None, arith=None):
    """the background network: rgb_raw [N, 3], density [N] and A_rgb, A_density (torch.nn.Linear layout, trunk layer 3 unrotated);
    z_density: the density's pre-activation"""
    dev = _dev(device)
    ar = arith or Exact()
    plan = Plan(pos, scale, shift, lattice.shape[1]).to(dev)
    feat, A, _, _ = features_bound(plan, lattice.detach().to(dev).double(), pos.detach().to(dev).double(), window, points_scaling)
    layers = _dev_layers(W, b, dev)
    z, Az, _, _ = chain_bound(ar, layers[:4], feat, A)
    z0 = z[:, 0].double()
    density = torch.nn.functional.softplus(z0)
    A_density = torch.sigmoid(z0) * Az[:, 0]
    sh = (sh if sh is not None else sh_fp32(dirs, 4)).to(dev)
    a, d1 = ar.gelu(z[:, 1:65])
    x = torch.cat([a, sh.to(a.dtype)], 1)
    Ax = torch.cat([((d1 * Az[:, 1:65]) ** 2 + a.double() ** 2).sqrt(), sh.abs()], 1)
    zr, Azr, _, _ = chain_bound(ar, layers[4:], x, Ax, first=4)
    return dict(rgb_raw=zr.double(), density=density, A_rgb=Azr, A_density=A_density, z_density=z0)
