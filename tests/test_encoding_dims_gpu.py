"""The permutohedral encoding kernels at every supported input width D in {2..6} and feature count F in {1, 2, 4, 8}, against the CPU
oracle (oracle/encoding_oracle.py) and against structural facts that need no oracle.

The image fit at the end is the end-to-end check: PermutoEncoding(2, 2^18, 16, F) + Linear(16 F, 64) ReLU Linear(64, 3), Adam at 1e-2,
500 full-batch steps on a procedural 512 x 512 RGB image. On an H100 80GB HBM3 (700 W power limit) it reached 47.0 dB (F = 2) and
49.5 dB (F = 4); the bar is 44 dB."""
import math

import numpy as np
import pytest
import torch

from oracle import encoding_oracle as eo

pytestmark = pytest.mark.gpu

PAIRS = [(D, F) for D in range(2, 7) for F in (1, 2, 4, 8)]
GUARD = 3                       # rows of sentinel before and after every C-ABI output
SENTINEL = -1234.5


def rel_err(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def make(D, F, L, T, concat=False, scaling=1e-3, seed=0, init_scale=1.0):
    import permutohedral_encoding as pe
    torch.manual_seed(seed)
    return pe.PermutoEncoding(D, T, L, F, np.geomspace(1.0, 1e-4, num=L), appply_random_shift_per_level=True, concat_points=concat,
                              concat_points_scaling=scaling, init_scale=init_scale)


def consts(enc):
    return enc.scale_factor.cpu(), enc.random_shift_per_level.detach().cpu()


def guarded(rows, cols):
    """a [rows, cols] view into a buffer with GUARD sentinel rows on each side"""
    buf = torch.full((rows + 2 * GUARD, cols), SENTINEL, device="cuda")
    return buf, buf[GUARD:GUARD + rows]


def guards_intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[buf.shape[0] - GUARD:] == SENTINEL).all())


def abi_args(enc, N, pos, window):
    D, L, F, T = enc.pos_dim, enc.nr_levels, enc.nr_feat_per_level, enc.capacity
    return (N, D, L, F, T, pos, enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(), window,
            1 if enc.concat_points else 0, enc.concat_points_scaling)


# (N, L, T, concat, window): every N, L, capacity kind, concat and window choice appears
FWD_CASES = [(1, 1, 5003, False, None), (31, 8, 2 ** 18, True, 0.6), (33, 32, 5003, True, None), (4097, 8, 5003, False, 0.6),
             (4097, 32, 2 ** 18, True, 0.6), (4097, 1, 2 ** 18, True, None)]


@pytest.mark.parametrize("D,F", PAIRS)
def test_forward_matches_oracle(cuda, D, F):
    from permuto_sdf_b200 import call
    for i, (N, L, T, concat, t) in enumerate(FWD_CASES):
        enc = make(D, F, L, T, concat, seed=i)
        torch.manual_seed(100 + i)
        pos = torch.rand(N, D) - 0.5
        window = None if t is None else eo.coarse2fine(L, t)
        sc, sh = consts(enc)
        ref = eo.encode(pos, enc.lattice_values.detach().cpu(), sc, sh, window, concat, 1e-3)
        out = enc(pos.cuda(), None if window is None else window.cuda())
        assert out.shape == ref.shape == (N, enc.output_dims())
        assert rel_err(out, ref) < 1e-5, (N, L, T, concat, t)
        buf, dst = guarded(N, enc.output_dims())
        win = torch.ones(L, device="cuda") if window is None else window.cuda()
        call("psdf_enc_forward", *abi_args(enc, N, pos.cuda(), win), dst)
        assert guards_intact(buf), "forward wrote outside its [N, C] block"
        assert torch.equal(dst, out)


@pytest.mark.parametrize("D,F", PAIRS)
def test_hashed_indices_exact(cuda, D, F):
    """the lattice gradient of sum(level columns) is the bary-weighted histogram of the hashed rows, in every feature column"""
    from permuto_sdf_b200 import call
    L, T, N = 4, 2 ** 16, 20000
    enc = make(D, F, L, T, seed=5)
    torch.manual_seed(2)
    pos = torch.rand(N, D) - 0.5
    sc, sh = consts(enc)
    idx = eo.all_indices(pos, sc, sh, T)
    g_l = torch.zeros(L, T, F, device="cuda")
    call("psdf_enc_backward", *abi_args(enc, N, pos.cuda(), torch.ones(L, device="cuda")), torch.ones(N, L * F, device="cuda"), g_l,
         None)
    expect_all = torch.zeros(L, T, dtype=torch.bool)
    expect_sig = torch.zeros(L, T, dtype=torch.bool)
    for l in range(L):
        _, _, bary = eo.simplex(pos, sc[l], sh[l])
        expect_all[l][idx[:, l].reshape(-1)] = True
        expect_sig[l][idx[:, l][bary.abs() > 1e-6]] = True
    assert int(expect_sig.sum()) > 1000
    for k in range(F):
        touched = (g_l[:, :, k] != 0).cpu()
        assert not bool((touched & ~expect_all).any()), "column %d: a row the oracle never hashes to" % k
        assert not bool((expect_sig & ~touched).any()), "column %d: a row the oracle hashes to is missing" % k
        assert torch.allclose(g_l[:, :, k], g_l[:, :, 0], rtol=1e-5), "every feature column gets the same histogram"


@pytest.mark.parametrize("D,F", PAIRS)
def test_constant_table_and_vertex_hit(cuda, D, F):
    L, T = 6, 4099
    enc = make(D, F, L, T, seed=7)
    window = eo.coarse2fine(L, 0.55)
    pos = torch.rand(500, D, device="cuda") - 0.5
    with torch.no_grad():
        enc.lattice_values.fill_(0.75)
        out = enc(pos, window.cuda())
    expect = (0.75 * window).repeat_interleave(F)[None].expand(500, -1)
    assert torch.allclose(out.cpu(), expect, rtol=1e-5, atol=1e-6)
    # a point on a lattice vertex of level 0 (no shift) returns that vertex's row: the nearest row of the table, at distance ~0
    with torch.no_grad():
        enc.lattice_values.uniform_(-1.0, 1.0)
        enc.random_shift_per_level.zero_()
    E = np.zeros((D + 1, D))
    E[0, :] = 1.0
    for i in range(1, D + 1):
        E[i, i:] = 1.0
        E[i, i - 1] = -float(i)
    target = np.zeros(D + 1)
    target[0], target[-1] = D + 1, -(D + 1)
    cf = np.linalg.lstsq(E, target, rcond=None)[0]
    p = torch.from_numpy(cf / enc.scale_factor[0].double().cpu().numpy()).float()[None].cuda()
    with torch.no_grad():
        row = enc(p)[0, :F]
    dist = (enc.lattice_values.detach()[0] - row[None]).abs().max(1).values
    assert float(dist.min()) < 1e-4 * float(row.abs().max())


def tiny_head_loss(encode_fn, lattice, p, Wm, proj, dev):
    p = p.clone().requires_grad_(True)
    feat = encode_fn(p)
    y = torch.tanh(feat @ Wm.to(dev)).sum(1, keepdim=True)
    (gp,) = torch.autograd.grad(y, p, torch.ones_like(y), create_graph=True)
    loss = (y ** 2).mean() + ((gp.norm(dim=1) - 1.0) ** 2).mean() + (gp * proj.to(dev)).sum(1).mean()
    (gl,) = torch.autograd.grad(loss, lattice, retain_graph=True)
    return y, gp, gl, loss


@pytest.mark.parametrize("D,F", PAIRS)
def test_backward_and_double_backward(cuda, D, F):
    from permuto_sdf_b200 import call
    N, L, T = 3000, 8, 5003
    enc = make(D, F, L, T, True, 0.5, seed=3)
    torch.manual_seed(4)
    pos = torch.rand(N, D) - 0.5
    window = eo.coarse2fine(L, 0.6)
    C = enc.output_dims()
    sc, sh = consts(enc)
    lat_cpu = enc.lattice_values.detach().cpu().clone().requires_grad_(True)
    # end to end through autograd: the tiny-head loss of test_encoding_gpu.py
    Wm, proj = torch.randn(C, 5) * 0.5, torch.randn(N, D)
    y0, gp0, gl0, loss0 = tiny_head_loss(lambda p: eo.encode(p, lat_cpu, sc, sh, window, True, 0.5), lat_cpu, pos, Wm, proj, "cpu")
    y1, gp1, gl1, loss1 = tiny_head_loss(lambda p: enc(p, window.cuda()), enc.lattice_values, pos.cuda(), Wm, proj, "cuda")
    assert rel_err(y1, y0) < 1e-4
    assert rel_err(gp1, gp0) < 1e-3, "positions gradient"
    assert abs(float(loss1.detach()) - float(loss0.detach())) / abs(float(loss0.detach())) < 1e-3
    assert rel_err(gl1, gl0) < 1e-3, "lattice gradient through value + double backward"
    # every backward and double-backward instantiation through the C ABI
    g_out, gg = torch.randn(N, C), torch.randn(N, D)
    p = pos.clone().requires_grad_(True)
    go = g_out.clone().requires_grad_(True)
    feat = eo.encode(p, lat_cpu, sc, sh, window, True, 0.5)
    ref_gl, ref_gp = torch.autograd.grad(feat, (lat_cpu, p), go, create_graph=True)
    ref_dl, ref_dgo = torch.autograd.grad((ref_gp * gg).sum(), (lat_cpu, go))
    args = abi_args(enc, N, pos.cuda(), window.cuda())
    for want_l, want_p in ((True, False), (False, True), (True, True)):
        g_l = torch.zeros(L, T, F, device="cuda") if want_l else None
        g_p = torch.full((N, D), SENTINEL, device="cuda") if want_p else None
        call("psdf_enc_backward", *args, g_out.cuda(), g_l, g_p)
        if want_l:
            assert rel_err(g_l, ref_gl) < 1e-3, "lattice gradient"
        if want_p:
            assert rel_err(g_p, ref_gp) < 1e-3, "positions gradient"
    for want_l, want_go in ((True, False), (False, True), (True, True)):
        g_l = torch.zeros(L, T, F, device="cuda") if want_l else None
        buf, g_go = guarded(N, C) if want_go else (None, None)
        call("psdf_enc_double_backward", *args, gg.cuda(), g_out.cuda(), g_l, g_go)
        if want_l:
            assert rel_err(g_l, ref_dl) < 1e-3, "double backward: lattice"
        if want_go:
            assert rel_err(g_go, ref_dgo) < 1e-3, "double backward: grad_out"
            assert guards_intact(buf)


@pytest.mark.parametrize("D", range(2, 7))
@pytest.mark.parametrize("F", (1, 4, 8))
def test_warp_aggregation(cuda, D, F):
    """all 32 lanes of a warp on one point, then pairs of lanes on one point: the peer sums must give the oracle's lattice gradient"""
    from permuto_sdf_b200 import call
    L, T = 4, 4099
    enc = make(D, F, L, T, seed=11)
    sc, sh = consts(enc)
    torch.manual_seed(12)
    base = torch.rand(64, D) - 0.5
    for pos in (base[:1].repeat(96, 1), base.repeat_interleave(2, 0)):
        N = pos.shape[0]
        g_out = torch.randn(N, L * F)
        lat = enc.lattice_values.detach().cpu().clone().requires_grad_(True)
        (ref,) = torch.autograd.grad(eo.encode(pos, lat, sc, sh), lat, g_out)
        g_l = torch.zeros(L, T, F, device="cuda")
        call("psdf_enc_backward", *abi_args(enc, N, pos.cuda(), torch.ones(L, device="cuda")), g_out.cuda(), g_l, None)
        assert rel_err(g_l, ref) < 1e-5


def test_largest_shared_memory_case(cuda):
    """D = 6, F = 8, L = 32 with concat: 66 KB of dynamic shared memory in the double backward"""
    from permuto_sdf_b200 import call
    D, F, L, T, N = 6, 8, 32, 2 ** 14, 1000
    enc = make(D, F, L, T, True, 0.5, seed=13)
    assert enc.output_dims() == 33 * 8
    sc, sh = consts(enc)
    torch.manual_seed(14)
    pos = torch.rand(N, D) - 0.5
    window = eo.coarse2fine(L, 0.8)
    C = enc.output_dims()
    g_out, gg = torch.randn(N, C), torch.randn(N, D)
    lat = enc.lattice_values.detach().cpu().clone().requires_grad_(True)
    p = pos.clone().requires_grad_(True)
    go = g_out.clone().requires_grad_(True)
    feat = eo.encode(p, lat, sc, sh, window, True, 0.5)
    ref_gl, ref_gp = torch.autograd.grad(feat, (lat, p), go, create_graph=True)
    ref_dl, ref_dgo = torch.autograd.grad((ref_gp * gg).sum(), (lat, go))
    args = abi_args(enc, N, pos.cuda(), window.cuda())
    out = torch.empty(N, C, device="cuda")
    call("psdf_enc_forward", *args, out)
    assert rel_err(out, feat) < 1e-5
    g_l, g_p = torch.zeros(L, T, F, device="cuda"), torch.empty(N, D, device="cuda")
    call("psdf_enc_backward", *args, g_out.cuda(), g_l, g_p)
    assert rel_err(g_l, ref_gl) < 1e-3 and rel_err(g_p, ref_gp) < 1e-3
    d_l, d_go = torch.zeros(L, T, F, device="cuda"), torch.empty(N, C, device="cuda")
    call("psdf_enc_double_backward", *args, gg.cuda(), g_out.cuda(), d_l, d_go)
    assert rel_err(d_l, ref_dl) < 1e-3 and rel_err(d_go, ref_dgo) < 1e-3


@pytest.mark.parametrize("D,F", [(1, 2), (7, 2), (3, 3), (3, 16)])
def test_unsupported_pairs_are_refused(cuda, D, F):
    from permuto_sdf_b200 import call
    enc = make(D, F, 4, 1024, True, seed=0)
    pos = torch.rand(40, D, device="cuda")
    with pytest.raises(RuntimeError) as e:
        enc(pos)
    assert "pos_dim=%d" % D in str(e.value) and "nr_feat_per_level=%d" % F in str(e.value)
    C = enc.output_dims()
    args = abi_args(enc, 40, pos, torch.ones(4, device="cuda"))
    out = torch.full((40, C), SENTINEL, device="cuda")
    g_l = torch.full((4, 1024, F), SENTINEL, device="cuda")
    g_p = torch.full((40, D), SENTINEL, device="cuda")
    with pytest.raises(RuntimeError):
        call("psdf_enc_forward", *args, out)
    with pytest.raises(RuntimeError):
        call("psdf_enc_backward", *args, torch.ones(40, C, device="cuda"), g_l, g_p)
    with pytest.raises(RuntimeError):
        call("psdf_enc_double_backward", *args, g_p.clone(), torch.ones(40, C, device="cuda"), g_l, out)
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all()) and bool((g_l == SENTINEL).all()) and bool((g_p == SENTINEL).all())


@pytest.mark.parametrize("D,F", [(2, 1), (6, 8)])
def test_cpu_tensors_are_refused(cuda, D, F):
    enc = make(D, F, 4, 1024)
    with pytest.raises(RuntimeError):
        enc(torch.rand(10, D))


def procedural_image(n=512):
    y, x = torch.meshgrid(torch.linspace(0, 1, n), torch.linspace(0, 1, n), indexing="ij")
    r = 0.5 + 0.5 * torch.sin(12 * x + 4 * torch.sin(7 * y))
    g = 0.5 + 0.5 * torch.cos(18 * y) * torch.sin(9 * x)
    disk = (((x - 0.6) ** 2 + (y - 0.4) ** 2) < 0.06).float()
    b = 0.3 * disk + 0.7 * (0.5 + 0.5 * torch.sin(30 * (x + y)))
    return torch.stack([r, g, b], -1).reshape(-1, 3), torch.stack([x, y], -1).reshape(-1, 2) - 0.5


def fit_image(F, steps=500):
    import permutohedral_encoding as pe
    torch.manual_seed(0)
    rgb, xy = procedural_image()
    rgb, xy = rgb.cuda(), xy.cuda()
    L = 16
    enc = pe.PermutoEncoding(2, 2 ** 18, L, F, np.geomspace(1.0, 2e-3, num=L))
    mlp = torch.nn.Sequential(torch.nn.Linear(L * F, 64), torch.nn.ReLU(), torch.nn.Linear(64, 3)).cuda()
    opt = torch.optim.Adam(list(enc.parameters()) + list(mlp.parameters()), lr=1e-2)
    for _ in range(steps):
        opt.zero_grad(set_to_none=True)
        loss = ((mlp(enc(xy)) - rgb) ** 2).mean()
        loss.backward()
        opt.step()
    with torch.no_grad():
        mse = float(((mlp(enc(xy)).clamp(0, 1) - rgb) ** 2).mean())
    return -10.0 * math.log10(mse)


@pytest.mark.parametrize("F", (2, 4))
def test_image_fit(cuda, F):
    psnr = fit_image(F)
    print("image fit, F = %d: %.2f dB" % (F, psnr))
    assert psnr > 44.0
