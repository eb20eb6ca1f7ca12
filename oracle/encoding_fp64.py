"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

fp64 reference of the stand-alone permutohedral encoding kernels (csrc/encoding.cu) at every input width D and feature count F: the
forward, the backward to the lattice and to the positions, and the double backward (to the lattice and to the upstream gradient),
each output with the error scale A its fp32 rounding error is proportional to, so that a kernel is judged per element.

The discrete decisions (remainder-0 point, rank, hashed rows) and the barycentric weights B are taken in fp32 from encoding_oracle
through backward_fp64.Plan: the kernels take the same decisions from the same fp32 operations, and their weights are those bits
(tests/test_encoding_fp64_gpu.py checks it on table entries with a single contribution). Everything downstream is fp64. The
derivative of B_r with respect to the scaled coordinates cf is the exact one inside the simplex of the rank:

    dB_r / dcf_j = sum_i M_ij (s(r = D - rank_i) - s(r = D + 1 - rank_i)) / (D + 1),   slot D + 1 folded into slot 0,

with M the elevation matrix (E = M cf; E_0 = sum_k cf_k, E_i = sum_{k >= i} cf_k - i cf_{i-1}). dB/dx_j = scale_j dB/dcf_j.

Error scales A (the sum of the absolute values of the terms an output is formed from, in the order the kernels form it):
  * forward feature (l, k): w_l sum_r |B_r| |v_rk|; concat column: |x_j s|; pad column: 0;
  * positions gradient j: sum_l w_l scale_lj sum_r (sum_k |v_rk| |g_lk|) K_rj + |g_cj s|, where K_rj = sum_i |M_ij| (s(r = D - rank_i)
    + s(r = D + 1 - rank_i)) / (D + 1) >= |dB_r / dcf_j|. The kernels do not form dB_r / dcf_j: they scatter the per-vertex products
    dB_r to the elevated coordinates and run the elevation backwards, so a coefficient that cancels exactly (e.g. d(E_0 - E_1)/dcf_1
    = 0) still has rounding error in the partial sums. K covers those partial sums;
  * grad_grad_out (l, k): w_l sum_r |v_rk| sum_j K_rj scale_lj |gg_j|; concat column: |gg_j s|; pad column: 0;
  * lattice gradient per table entry e: the value (prefill + contributions), n_e = the number of (sample, vertex) contributions and
    A_e = sum |contribution| (backward: w_l |B_r| |g_lk|; double backward: w_l sum_j K_rj scale_lj |gg_j| |g_lk|).

EPS, from the kernels' fp32 arithmetic (u = 2^-24; a chain of n roundings on partial sums bounded by A errs by <= n u A):
  * forward: wr = B_r w (1) and an fma chain over D + 1 vertices (D + 1): D + 2 <= 8 roundings; without fma (products, then a sum,
    as the fp32 oracle forms it) 2 D + 3 <= 15 -> EPS_FWD = 32 u = 2^-19;
  * positions gradient: the dot over F features (F), times w (1), bary_grad_to_cf (dB_{D+1} += dB_0, a - b, times 1/(D+1), the
    running sum over D, the product and difference with (k + 1) de_{k+1}: D + 5), the fma with scale (1), the level loop of a group
    (L / 4 <= 8 levels), the sum of the 4 groups (3) and the concat fma (1): F + D + 19 <= 33 -> EPS_POS = 64 u = 2^-18;
  * grad_grad_out: dcf = u scale (1), the elevation of the direction (D + 2), bary_tangent (1/(D+1), the +- scatter, the fold: 4),
    db w (1), an fma chain over D + 1 vertices: 2 D + 9 <= 21 -> EPS_GGO = 32 u = 2^-19;
  * lattice gradient, float: each contribution is formed with M_LAT = 2 roundings (B w, then g) and the n_e additions (warp peer
    sums, vector atomics, the prefill) each round once: |got - ref| <= (n_e + M_LAT) u (A_e + |prefill|), up to a slack for the first
    order. The double backward's contributions carry the tangent chain above, M_DLAT = D + 9 <= 16 roundings;
  * lattice gradient, fixed point: each contribution is rounded to the 2^-34 grid once (<= 2^-35) after its fp32 product chain
    (M u |c|); the flush converts the integer total to fp32 (u |total|) and adds it to the prefill (u |ref|).
Every EPS is far below the 1e-3 ceiling of the tensor-wide ratio. tests/test_encoding_fp64_reference_cpu.py shows that fp32
arithmetic (the fp32 oracle and its autograd) stays within EPS A / 4 and that a bf16 table or a dropped vertex breaks EPS A.
"""
import numpy as np
import torch

from . import backward_fp64 as R

F64 = torch.float64
U = 2.0 ** -24
EPS_FWD = 32 * U
EPS_POS = 64 * U
EPS_GGO = 32 * U
M_LAT = 2
M_DLAT = 16
FX_STEP = 2.0 ** -35


def n_extra(D, F, concat):
    """concat columns: E = ceil(D / F) groups of F"""
    return (D + F - 1) // F * F if concat else 0


def elevation_matrix(D, dtype=F64, device=None):
    """M [D+1, D]: elevated = M cf"""
    M = torch.zeros(D + 1, D, dtype=dtype, device=device)
    M[0, :] = 1.0
    for i in range(1, D + 1):
        M[i, i:] = 1.0
        M[i, i - 1] = -float(i)
    return M


def bary_coefficients(rank, D):
    """exact dB_r / dcf_j [N, D+1, D] of the simplex of `rank`, and K [N, D+1, D] (see the module docstring)"""
    N = rank.shape[0]
    dev = rank.device
    M = elevation_matrix(D, device=dev)
    up = torch.zeros(N, D + 1, D + 2, dtype=F64, device=dev).scatter_(2, (D - rank)[:, :, None], 1.0)
    dn = torch.zeros(N, D + 1, D + 2, dtype=F64, device=dev).scatter_(2, (D + 1 - rank)[:, :, None], 1.0)

    def fold(P):
        P = P.clone()
        P[:, :, 0] += P[:, :, D + 1]
        return P[:, :, :D + 1]
    coef = torch.einsum("nir,ij->nrj", fold(up) - fold(dn), M) / (D + 1)
    K = torch.einsum("nir,ij->nrj", fold(up) + fold(dn), M.abs()) / (D + 1)
    return coef, K


def plan_of(pos, scale, shift, T, device=None):
    """discrete decisions and fp32 weights (backward_fp64.Plan), plus the per-level weight derivatives, on `device`"""
    plan = R.Plan(pos, scale, shift, T)
    dev = torch.device(device) if device is not None else torch.device("cpu")
    plan.to(dev)
    plan.coef, plan.K = [], []
    for l in range(plan.L):
        c, K = bary_coefficients(plan.rank[l], plan.D)
        plan.coef.append(c)
        plan.K.append(K)
    return plan


def _f32(x):
    return float(np.float32(x))


def reference(plan, lattice, window, concat, scaling, g_out=None, gg=None, pos=None, prefill=None, prefill2=None):
    """-> dict of fp64 tensors on the plan's device:
    out, A_out [N, C]; with g_out: pos_grad, A_pos [N, D]; lat, lat_A, lat_n [L, T, F] (lat includes `prefill`, A excludes it);
    with gg: ggo, A_ggo [N, C]; with g_out and gg: dlat, dlat_A, dlat_n (dlat includes `prefill2`).
    pos: the fp32 positions (for the concat columns); window: [L] fp32 (None: ones); scaling: rounded to fp32 as the kernels take it."""
    dev = plan.bary[0].device
    L, T, N, D = plan.L, plan.T, plan.N, plan.D
    F = lattice.shape[2]
    lat64 = lattice.detach().to(dev).double()
    w = window.detach().to(dev).double() if window is not None else torch.ones(L, dtype=F64, device=dev)
    s = _f32(scaling)
    EF = n_extra(D, F, concat)
    C = L * F + EF
    x = pos.detach().to(dev).double() if pos is not None else None
    go = g_out.detach().to(dev).double() if g_out is not None else None
    u = gg.detach().to(dev).double() if gg is not None else None
    out = torch.zeros(N, C, dtype=F64, device=dev)
    A_out = torch.zeros_like(out)
    r = dict(out=out, A_out=A_out)
    if go is not None:
        pg, A_pg = torch.zeros(N, D, dtype=F64, device=dev), torch.zeros(N, D, dtype=F64, device=dev)
        lat = prefill.detach().to(dev).double().clone() if prefill is not None else torch.zeros(L, T, F, dtype=F64, device=dev)
        lat_A, lat_n = torch.zeros(L, T, F, dtype=F64, device=dev), torch.zeros(L, T, dtype=F64, device=dev)
    if u is not None:
        ggo, A_ggo = torch.zeros(N, C, dtype=F64, device=dev), torch.zeros(N, C, dtype=F64, device=dev)
        if go is not None:
            dlat = prefill2.detach().to(dev).double().clone() if prefill2 is not None else torch.zeros(L, T, F, dtype=F64, device=dev)
            dlat_A = torch.zeros(L, T, F, dtype=F64, device=dev)
    for l in range(L):
        idx = plan.idx[l]                                     # [N, D+1]
        flat = idx.reshape(-1)
        vals = lat64[l][idx]                                  # [N, D+1, F]
        B = plan.bary[l]
        sc = plan.scale[l]
        out[:, l * F:(l + 1) * F] = w[l] * (B[:, :, None] * vals).sum(1)
        A_out[:, l * F:(l + 1) * F] = w[l] * (B.abs()[:, :, None] * vals.abs()).sum(1)
        dBdx = plan.coef[l] * sc                              # [N, D+1, D]
        Kx = plan.K[l] * sc
        if go is not None:
            g = go[:, l * F:(l + 1) * F]
            dot = (vals * g[:, None, :]).sum(2)               # [N, D+1]
            adot = (vals.abs() * g.abs()[:, None, :]).sum(2)
            pg += w[l] * (dot[:, :, None] * dBdx).sum(1)
            A_pg += w[l] * (adot[:, :, None] * Kx).sum(1)
            c = w[l] * B[:, :, None] * g[:, None, :]          # [N, D+1, F]
            lat[l].index_add_(0, flat, c.reshape(-1, F))
            lat_A[l].index_add_(0, flat, c.abs().reshape(-1, F))
            lat_n[l].index_add_(0, flat, torch.ones_like(flat, dtype=F64))
        if u is not None:
            dB = (dBdx * u[:, None, :]).sum(2)                 # [N, D+1]: tangent of the weights along gg
            adB = (Kx * u.abs()[:, None, :]).sum(2)
            ggo[:, l * F:(l + 1) * F] = w[l] * (dB[:, :, None] * vals).sum(1)
            A_ggo[:, l * F:(l + 1) * F] = w[l] * (adB[:, :, None] * vals.abs()).sum(1)
            if go is not None:
                g = go[:, l * F:(l + 1) * F]
                dlat[l].index_add_(0, flat, (w[l] * dB[:, :, None] * g[:, None, :]).reshape(-1, F))
                dlat_A[l].index_add_(0, flat, (w[l] * adB[:, :, None] * g.abs()[:, None, :]).reshape(-1, F))
    if concat:
        base = L * F
        out[:, base:base + D] = x * s
        A_out[:, base:base + D] = (x * s).abs()
        if go is not None:
            pg += go[:, base:base + D] * s
            A_pg += (go[:, base:base + D] * s).abs()
        if u is not None:
            ggo[:, base:base + D] = u * s
            A_ggo[:, base:base + D] = (u * s).abs()
    if go is not None:
        r.update(pos_grad=pg, A_pos=A_pg, lat=lat, lat_A=lat_A, lat_n=lat_n[:, :, None].expand(L, T, F))
    if u is not None:
        r.update(ggo=ggo, A_ggo=A_ggo)
        if go is not None:
            r.update(dlat=dlat, dlat_A=dlat_A, dlat_n=r["lat_n"])
    return r


def lattice_bound(ref, A, n, prefill, m):
    """per-entry bound of a float lattice gradient (module docstring); prefill: the values the table held before the call"""
    P = prefill.double().abs() if prefill is not None else 0.0
    return (n + m) * U * (A + P) * (1.0 + 2.0 ** -8)


def lattice_bound_fx(ref, A, n, m):
    """per-entry bound of a fixed-point lattice gradient (ref includes the prefill)"""
    return (n * FX_STEP + (m + 1) * U * A + U * ref.abs()) * (1.0 + 2.0 ** -8)


def encode_st(pos64, lattice64, plan, window, F, concat, scaling):
    """differentiable fp64 encoding at any F: value = the fp32 barycentric weights, position derivative = the exact one
    (straight-through, as backward_fp64.encode_st), concat columns in E = ceil(D / F) groups of F"""
    cols = []
    w = window.double().to(pos64.device) if window is not None else torch.ones(plan.L, dtype=F64, device=pos64.device)
    for l in range(plan.L):
        cf = (pos64 + plan.shift[l]) * plan.scale[l]
        lin = R.bary_linear(cf, plan.rank[l], plan.rem0[l])
        B = plan.bary[l] + (lin - lin.detach())
        cols.append(w[l] * (B[:, :, None] * lattice64[l][plan.idx[l]]).sum(1))
    if concat:
        N, D = pos64.shape
        cols.append(pos64 * _f32(scaling))
        pad = n_extra(D, F, concat) - D
        if pad:
            cols.append(torch.zeros(N, pad, dtype=F64, device=pos64.device))
    return torch.cat(cols, 1)


def worst(err, bound):
    """max of err / bound, where a zero bound admits only a zero error"""
    err, bound = err.double(), bound.double()
    ok0 = (bound == 0) & (err == 0)
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)), torch.full_like(err, float("inf")))
    ratio = torch.where(ok0, torch.zeros_like(ratio), ratio)
    return float(ratio.max()) if ratio.numel() else 0.0
