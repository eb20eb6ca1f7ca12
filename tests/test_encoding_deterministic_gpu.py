"""The deterministic lattice gradient of the permutohedral encoding (psdf_enc_backward_fx, psdf_enc_double_backward_fx and
PermutoEncoding(deterministic=True)) at every supported (D, F) pair, with and without concat columns, under a coarse-to-fine window
with some levels partly open and some closed.

The rows are clustered (a few hundred centres, exact duplicate rows, sorted by centre), and the level scales run from 1 to 1e-3, so
whole warps share vertices on the coarse levels and neighbouring warps of a block share them on the fine ones. The reference values
come from the CPU oracle (oracle/encoding_oracle.py): its fp32 simplex reproduces the kernels' vertices, and the gradients are summed
from its weights in fp64."""
import numpy as np
import pytest
import torch

from oracle import encoding_oracle as eo

pytestmark = pytest.mark.gpu

PAIRS = [(D, F) for D in range(2, 7) for F in (1, 2, 4, 8)]
N, L, T = 40003, 8, 2 ** 14          # N: a partial last warp
SENTINEL = -1234.5
SIGMAS = np.geomspace(1.0, 1e-3, num=L)


def make(D, F, L=L, T=T, concat=False, seed=0, deterministic=True):
    import permutohedral_encoding as pe
    torch.manual_seed(seed)
    return pe.PermutoEncoding(D, T, L, F, SIGMAS if L == len(SIGMAS) else np.geomspace(1.0, 1e-3, num=L), appply_random_shift_per_level=True, concat_points=concat,
                              concat_points_scaling=0.5, init_scale=1.0, deterministic=deterministic)


def clustered(D, n, seed):
    """n rows around 300 centres, sorted by centre, with exact duplicate rows"""
    g = torch.Generator().manual_seed(seed)
    centres = torch.rand(300, D, generator=g) - 0.5
    cid = torch.randint(0, 300, (n,), generator=g).sort().values
    pos = centres[cid] + 2e-3 * torch.randn(n, D, generator=g)
    pos[n // 2:n // 2 + n // 8] = pos[:n // 8]
    pos[n - 50:] = pos[n - 100:n - 50]
    return pos


def abi_args(enc, pos, window):
    return (pos.shape[0], enc.pos_dim, enc.nr_levels, enc.nr_feat_per_level, enc.capacity, pos, enc.lattice_values.detach(),
            enc.scale_factor, enc.shift_tensor(), window, 1 if enc.concat_points else 0, enc.concat_points_scaling)


WINDOW = eo.coarse2fine(L, 0.55)       # levels 0..3 open, 4 partly, 5..7 closed
OPEN = [l for l in range(L) if float(WINDOW[l]) > 0]
_GEOMETRY = {}


def geometry(D):
    """positions, gg, shifts, and per open level the oracle's vertex rows, weights and weight tangents along gg; the same for every F
    and concat choice at this D (the CPU oracle is the slow part of these tests)"""
    if D not in _GEOMETRY:
        g = torch.Generator().manual_seed(D)
        pos, gg, shift = clustered(D, N, D), torch.randn(N, D, generator=g), torch.randn(L, D, generator=g) * 10
        sc = eo.scale_factor(SIGMAS, D)
        levels = []
        for l in OPEN:
            p = pos.clone().requires_grad_(True)
            rem0, rank, bary = eo.simplex(p, sc[l], shift[l])
            u = torch.zeros_like(bary, requires_grad=True)        # tangent along gg: d/du of <(d bary/d pos)^T u, gg>
            (gp,) = torch.autograd.grad(bary, p, u, create_graph=True)
            (db,) = torch.autograd.grad(gp, u, gg)
            levels.append((eo.vertex_indices(rem0, rank, T), bary.detach().double(), db.double()))
        _GEOMETRY[D] = (pos, gg, shift, levels)
    return _GEOMETRY[D]


class Case:
    def __init__(self, D, F, concat, seed=0):
        from permuto_sdf_b200 import call
        self.call = call
        self.enc = make(D, F, concat=concat, seed=seed)
        self.D, self.F, self.C = D, F, self.enc.output_dims()
        self.window = WINDOW
        self.pos, self.gg, shift, self.levels = geometry(D)
        with torch.no_grad():
            self.enc.random_shift_per_level.copy_(shift)
        torch.manual_seed(seed + 1)
        self.g_out = torch.randn(N, self.C)
        self.ws = self.enc.fx_workspace(torch.device("cuda", 0))

    def bwd(self, fn, perm=None, lattice=True, want_pos=True, fx="ws"):
        pos, g_out = (self.pos, self.g_out) if perm is None else (self.pos[perm], self.g_out[perm])
        g_l = torch.zeros(L, T, self.F, device="cuda") if lattice is True else lattice
        g_p = torch.full((N, self.D), SENTINEL, device="cuda") if want_pos else None
        extra = () if fn == "psdf_enc_backward" else (self.ws if isinstance(fx, str) else fx,)
        self.call(fn, *abi_args(self.enc, pos.cuda(), self.window.cuda()), g_out.cuda(), g_l, g_p, *extra)
        return g_l, g_p

    def dbl(self, fn, perm=None, lattice=True, want_go=True, fx="ws"):
        pos, g_out, gg = (self.pos, self.g_out, self.gg) if perm is None else (self.pos[perm], self.g_out[perm], self.gg[perm])
        g_l = torch.zeros(L, T, self.F, device="cuda") if lattice is True else lattice
        g_go = torch.full((N, self.C), SENTINEL, device="cuda") if want_go else None
        extra = () if fn == "psdf_enc_double_backward" else (self.ws if isinstance(fx, str) else fx,)
        self.call(fn, *abi_args(self.enc, pos.cuda(), self.window.cuda()), gg.cuda(), g_out.cuda(), g_l, g_go, *extra)
        return g_l, g_go

    def workspace_clear(self):
        torch.cuda.synchronize()
        return int(self.ws.count_nonzero()) == 0

    def oracle(self, double):
        """fp64 lattice gradient, and per entry the number of contributions n_e and the sum of their magnitudes S_e (closed levels:
        no contributions)"""
        F = self.F
        ref, cnt, mag = (torch.zeros(L, T, F, dtype=torch.float64) for _ in range(3))
        for l, (idx, bary, db) in zip(OPEN, self.levels):
            a = (db if double else bary) * float(self.window[l])
            c = a[:, :, None] * self.g_out[:, None, l * F:(l + 1) * F].double()       # [N, D+1, F]
            flat = idx.reshape(-1)
            ref[l].index_add_(0, flat, c.reshape(-1, F))
            mag[l].index_add_(0, flat, c.abs().reshape(-1, F))
            cnt[l].index_add_(0, flat, torch.ones_like(c).reshape(-1, F))
        return ref, cnt, mag


def rel_err(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def check_against_float_and_oracle(fx, fl, ref, cnt, mag):
    assert rel_err(fx, ref) < 1e-3
    # each contribution is rounded to the 2^-34 grid once (<= 2^-35), the float path rounds each of its n_e - 1 additions, and the
    # flush rounds the total to fp32 once
    bound = cnt * 2.0 ** -35 + (cnt + 1) * 2.0 ** -24 * mag * 1.01
    diff = (fx.cpu().double() - fl.cpu().double()).abs()
    assert bool((diff <= bound).all()), float((diff - bound).max())
    assert bool((fx.cpu()[cnt == 0] == 0).all()), "an entry without contributions was written"


@pytest.mark.parametrize("concat", (False, True))
@pytest.mark.parametrize("D,F", PAIRS)
def test_backward_is_order_independent_and_accurate(cuda, D, F, concat):
    c = Case(D, F, concat, seed=D * 10 + F)
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(7))
    rev = torch.arange(N - 1, -1, -1)
    g_l, g_p = c.bwd("psdf_enc_backward_fx")
    assert c.workspace_clear()
    assert int((g_l != 0).sum()) > 200
    for gl2, _ in (c.bwd("psdf_enc_backward_fx", perm), c.bwd("psdf_enc_backward_fx", rev), c.bwd("psdf_enc_backward_fx"),
                   c.bwd("psdf_enc_backward_fx", perm, want_pos=False)):
        assert torch.equal(gl2, g_l)
        assert c.workspace_clear()
    fl_l, fl_p = c.bwd("psdf_enc_backward")
    assert torch.equal(g_p, fl_p), "positions gradient must be the float kernel's"
    ref, cnt, mag = c.oracle(double=False)
    check_against_float_and_oracle(g_l, fl_l, ref, cnt, mag)


@pytest.mark.parametrize("concat", (False, True))
@pytest.mark.parametrize("D,F", PAIRS)
def test_double_backward_is_order_independent_and_accurate(cuda, D, F, concat):
    c = Case(D, F, concat, seed=D * 10 + F + 100)
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(8))
    rev = torch.arange(N - 1, -1, -1)
    g_l, g_go = c.dbl("psdf_enc_double_backward_fx")
    assert c.workspace_clear()
    assert int((g_l != 0).sum()) > 200
    for gl2, _ in (c.dbl("psdf_enc_double_backward_fx", perm), c.dbl("psdf_enc_double_backward_fx", rev),
                   c.dbl("psdf_enc_double_backward_fx"), c.dbl("psdf_enc_double_backward_fx", perm, want_go=False)):
        assert torch.equal(gl2, g_l)
        assert c.workspace_clear()
    fl_l, fl_go = c.dbl("psdf_enc_double_backward")
    assert torch.equal(g_go, fl_go), "grad_grad_out must be the float kernel's"
    ref, cnt, mag = c.oracle(double=True)
    check_against_float_and_oracle(g_l, fl_l, ref, cnt, mag)


@pytest.mark.parametrize("D,F", PAIRS)
def test_call_contract(cuda, D, F):
    c = Case(D, F, True, seed=3)
    # a pre-filled grad_lattice is added to exactly once
    g_zero, _ = c.bwd("psdf_enc_backward_fx")
    pre = torch.randn(L, T, F, device="cuda")
    g_pre, _ = c.bwd("psdf_enc_backward_fx", lattice=pre.clone())
    assert torch.equal(g_pre, pre + g_zero)
    assert c.workspace_clear()
    d_zero, _ = c.dbl("psdf_enc_double_backward_fx")
    d_pre, _ = c.dbl("psdf_enc_double_backward_fx", lattice=pre.clone())
    assert torch.equal(d_pre, pre + d_zero)
    assert c.workspace_clear()
    # without grad_lattice: the float entry points, whatever fx_lattice is
    _, fl_p = c.bwd("psdf_enc_backward", lattice=None)
    for fx in ("ws", None):
        _, g_p = c.bwd("psdf_enc_backward_fx", lattice=None, fx=fx)
        assert torch.equal(g_p, fl_p)
    _, fl_go = c.dbl("psdf_enc_double_backward", lattice=None)
    for fx in ("ws", None):
        _, g_go = c.dbl("psdf_enc_double_backward_fx", lattice=None, fx=fx)
        assert torch.equal(g_go, fl_go)
    assert c.workspace_clear()
    # a lattice output without accumulators is refused before anything is written
    g_l = torch.full((L, T, F), SENTINEL, device="cuda")
    with pytest.raises(RuntimeError):
        c.bwd("psdf_enc_backward_fx", lattice=g_l, fx=None)
    with pytest.raises(RuntimeError):
        c.dbl("psdf_enc_double_backward_fx", lattice=g_l, fx=None)
    # accumulators on the CPU are refused
    with pytest.raises(RuntimeError):
        c.bwd("psdf_enc_backward_fx", fx=torch.zeros(L, T, F, dtype=torch.int64))
    torch.cuda.synchronize()
    assert bool((g_l == SENTINEL).all())


@pytest.mark.parametrize("D,F", [(1, 2), (7, 2), (3, 3), (3, 16)])
def test_unsupported_pairs_are_refused(cuda, D, F):
    from permuto_sdf_b200.permutohedral_encoding import _enc_call
    enc = make(D, F, 4, 1024, True)
    pos = torch.rand(40, D, device="cuda")
    with pytest.raises(RuntimeError) as e:
        enc(pos)
    assert "pos_dim=%d" % D in str(e.value) and "nr_feat_per_level=%d" % F in str(e.value)
    C = enc.output_dims()
    args = abi_args(enc, pos, torch.ones(4, device="cuda"))
    g_l = torch.full((4, 1024, F), SENTINEL, device="cuda")
    g_p = torch.full((40, D), SENTINEL, device="cuda")
    g_go = torch.full((40, C), SENTINEL, device="cuda")
    ws = enc.fx_workspace(pos.device)
    with pytest.raises(RuntimeError) as e:
        _enc_call("psdf_enc_backward_fx", enc, *args, torch.ones(40, C, device="cuda"), g_l, g_p, ws)
    assert "pos_dim=%d" % D in str(e.value) and "nr_feat_per_level=%d" % F in str(e.value)
    with pytest.raises(RuntimeError) as e:
        _enc_call("psdf_enc_double_backward_fx", enc, *args, g_p.clone(), torch.ones(40, C, device="cuda"), g_l, g_go, ws)
    assert "pos_dim=%d" % D in str(e.value) and "nr_feat_per_level=%d" % F in str(e.value)
    torch.cuda.synchronize()
    assert bool((g_l == SENTINEL).all()) and bool((g_p == SENTINEL).all()) and bool((g_go == SENTINEL).all())
    assert int(ws.count_nonzero()) == 0


@pytest.mark.parametrize("D,F", [(2, 1), (6, 8)])
def test_cpu_tensors_are_refused(cuda, D, F):
    enc = make(D, F, 4, 1024)
    with pytest.raises(RuntimeError):
        enc(torch.rand(10, D))


def train(D, F, orders, grad_in_place=False, steps=20, n=4099):
    """20 Adam steps of element-wise feature terms plus an eikonal term (no GEMM), every step's batch fed in the row order
    orders[step]; -> the final lattice_values"""
    enc = make(D, F, L=L, T=T, concat=True, seed=21)
    enc.lattice_values.data.mul_(1e-2)
    enc.grad_in_place = grad_in_place
    opt = torch.optim.Adam(enc.parameters(), lr=1e-3)
    coef = torch.linspace(-1.0, 1.0, enc.output_dims(), device="cuda")
    window = eo.coarse2fine(L, 0.55).cuda()
    for s in range(steps):
        pos = clustered(D, n, 100 + s)[orders[s]].cuda().requires_grad_(True)
        opt.zero_grad(set_to_none=False)
        feat = enc(pos, window)
        y = (feat * coef).sum(1)
        (gp,) = torch.autograd.grad(y, pos, torch.ones_like(y), create_graph=True)
        loss = ((feat - 0.1) ** 2).mean() + torch.sin(3 * feat).abs().mean() + ((gp.norm(dim=1) - 1.0) ** 2).mean()
        loss.backward()
        opt.step()
    return enc.lattice_values.detach().clone()


@pytest.mark.parametrize("D,F", PAIRS)
def test_training_is_independent_of_the_row_order(cuda, D, F):
    n = 4099
    gen = torch.Generator().manual_seed(D * 8 + F)
    a = [torch.randperm(n, generator=gen) for _ in range(20)]
    b = [torch.randperm(n, generator=gen) for _ in range(20)]
    la = train(D, F, a)
    assert float((la - make(D, F, concat=True, seed=21).lattice_values.detach() * 1e-2).abs().max()) > 0, "training moved nothing"
    assert torch.equal(train(D, F, b), la)
    assert torch.equal(train(D, F, a, grad_in_place=True), la)
