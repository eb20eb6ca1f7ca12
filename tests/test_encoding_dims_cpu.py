"""The permutohedral encoding at every input width from 2 to 6 and 1, 2, 4 or 8 features per level, without a GPU.

Known-answer tests of the CPU oracle (oracle/encoding_oracle.py) at D in {2, 5, 6} and F in {1, 4, 8}: partition of unity, vertex
hit, continuity across simplex faces, fp64 finite differences of the first and the double backward, the concat layout for F >= D and
F < D. Then a compile check of csrc/encoding.cu with the command `build()` uses: no k_enc_* instantiation spills, and the (3, 2) and
(4, 2) ones keep the register counts they had when the library was built for those two pairs only."""
import math
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from oracle import encoding_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
DIMS, FEATS = (2, 5, 6), (1, 4, 8)


def setup(D, F, L=3, T=2 ** 12, seed=0, dtype=torch.float32):
    torch.manual_seed(seed)
    scale = eo.scale_factor(np.geomspace(1.0, 1e-2, L), D)
    shift = torch.randn(L, D) * 10
    lattice = torch.randn(L, T, F)
    pos = (torch.rand(300, D) - 0.5).to(dtype)
    return pos, lattice, scale, shift


def elevation_matrix(D):
    """[D+1, D] matrix of the elevation: elevated[0] = sum_k cf[k]; elevated[i] = sum_{k >= i} cf[k] - i cf[i-1]"""
    E = np.zeros((D + 1, D))
    E[0, :] = 1.0
    for i in range(1, D + 1):
        E[i, i:] = 1.0
        E[i, i - 1] = -float(i)
    return E


@pytest.mark.parametrize("D", DIMS)
def test_partition_of_unity(D):
    pos, lattice, scale, shift = setup(D, 1)
    for l in range(scale.shape[0]):
        rem0, rank, bary = eo.simplex(pos, scale[l], shift[l])
        assert torch.allclose(bary.sum(1), torch.ones(pos.shape[0]), atol=1e-5)
        assert float(bary.min()) > -1e-5
        assert bool((rank.sort(1).values == torch.arange(D + 1)).all())      # rank is a permutation
        assert bool((rem0.sum(1) == 0).all()) and bool((rem0 % (D + 1) == 0).all())


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("F", FEATS)
def test_vertex_hit_returns_vertex_row(D, F):
    """a point whose elevated coordinates are a remainder-0 lattice point gets that vertex's row (weight 1)"""
    T = 2 ** 12
    scale = eo.scale_factor([1.0], D)
    shift = torch.zeros(1, D)
    lattice = torch.randn(1, T, F, dtype=torch.float64)
    target = np.zeros(D + 1)
    target[0], target[-1] = D + 1, -(D + 1)
    cf = np.linalg.lstsq(elevation_matrix(D), target, rcond=None)[0]
    pos = (torch.from_numpy(cf) / scale[0].double())[None]
    rem0, rank, bary = eo.simplex(pos, scale[0], shift[0])
    assert abs(float(bary.max()) - 1.0) < 1e-9
    out = eo.encode(pos, lattice, scale, shift)
    idx = eo.vertex_indices(rem0, rank, T)[0, int(bary.argmax(1))]
    assert out.shape == (1, F)
    assert torch.allclose(out[0], lattice[0, idx], atol=1e-9)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("F", FEATS)
def test_continuity_across_simplex_faces(D, F):
    pos, lattice, scale, shift = setup(D, F, seed=3)
    a = pos[:20].double()
    b = a + 0.05 * torch.nn.functional.normalize(pos[20:40].double(), dim=1)
    ts = torch.linspace(0, 1, 2000, dtype=torch.float64)[:, None, None]
    seg = (a[None] * (1 - ts) + b[None] * ts).reshape(-1, D)
    out = eo.encode(seg, lattice.double(), scale, shift).reshape(2000, 20, -1)
    assert float((out[1:] - out[:-1]).abs().max()) < 0.05, "features must be continuous along a segment"


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("F", FEATS)
def test_gradients_match_finite_differences_fp64(D, F):
    pos, lattice, scale, shift = setup(D, F, L=2, seed=5, dtype=torch.float64)
    lattice = lattice.double().requires_grad_(True)
    Wm = torch.randn(2 * F, 1, dtype=torch.float64)
    p = pos[:40].clone().requires_grad_(True)

    def f(pp, lat=lattice):
        return torch.tanh(eo.encode(pp, lat, scale, shift) @ Wm)
    (g,) = torch.autograd.grad(f(p).sum(), p, create_graph=True)
    eps = 1e-7
    for j in range(D):
        dp = torch.zeros_like(p)
        dp[:, j] = eps
        fd = (f(p + dp) - f(p - dp)) / (2 * eps)
        ok = (fd[:, 0] - g[:, j]).abs() < 1e-4 * (1 + g[:, j].abs())      # points next to a face may cross it
        assert ok.float().mean() > 0.9
    # double backward: d/d lattice of sum(g * v) against finite differences of the analytic gradient
    v = torch.randn_like(g)
    (gl,) = torch.autograd.grad((g * v).sum(), lattice)
    nz = gl.abs().reshape(-1).argmax()
    d = torch.zeros_like(lattice).reshape(-1)
    d[nz] = 1e-6
    d = d.reshape(lattice.shape)

    def grad_at(lat):
        pp = p.detach().clone().requires_grad_(True)
        return torch.autograd.grad(f(pp, lat).sum(), pp)[0]
    fd = ((grad_at(lattice.detach() + d) - grad_at(lattice.detach() - d)) * v).sum() / 2e-6
    assert abs(float(fd) - float(gl.reshape(-1)[nz])) < 1e-4 * (1 + abs(float(fd)))


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("F", FEATS)
def test_concat_layout(D, F):
    """E = ceil(D / F) column groups of F after the level columns: the D coordinates times the scaling, zeros past D"""
    pos, lattice, scale, shift = setup(D, F)
    L = scale.shape[0]
    E = int(math.ceil(D / F))
    out = eo.encode(pos, lattice, scale, shift, None, True, 1e-3)
    assert out.shape == (pos.shape[0], (L + E) * F)
    assert torch.allclose(out[:, L * F:L * F + D], pos * 1e-3)
    rest = out[:, L * F + D:]
    assert rest.numel() == 0 or float(rest.abs().max()) == 0.0
    assert E == (1 if F >= D else -(-D // F))


# ---------------------------------------------------------------------------------------------------------- compile check
# ptxas registers of the (3, 2) and (4, 2) kernels when the library was built for those two pairs only (CUDA 12.9, sm_90a)
PARENT_REGS = {
    "k_enc_forward<3, 2>": 46, "k_enc_forward<4, 2>": 54,
    "k_enc_backward<3, 2, false, true>": 48, "k_enc_backward<3, 2, true, false>": 45, "k_enc_backward<3, 2, true, true>": 64,
    "k_enc_backward<4, 2, false, true>": 56, "k_enc_backward<4, 2, true, false>": 46, "k_enc_backward<4, 2, true, true>": 80,
    "k_enc_double_backward<3, 2, false, true>": 48, "k_enc_double_backward<3, 2, true, false>": 48,
    "k_enc_double_backward<3, 2, true, true>": 56, "k_enc_double_backward<4, 2, false, true>": 48,
    "k_enc_double_backward<4, 2, true, false>": 40, "k_enc_double_backward<4, 2, true, true>": 56,
}


@pytest.fixture(scope="module")
def enc_kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("encoding.cu",)) if r["kernel"].startswith("k_enc_")}


def test_every_instantiation_is_built_without_spills(enc_kernels):
    expect = set()
    for D in range(2, 7):
        for F in (1, 2, 4, 8):
            expect.add("k_enc_forward<%d, %d>" % (D, F))
            for flags in ("false, true", "true, false", "true, true"):
                expect.add("k_enc_backward<%d, %d, %s>" % (D, F, flags))
                expect.add("k_enc_double_backward<%d, %d, %s>" % (D, F, flags))
    assert set(enc_kernels) == expect
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in enc_kernels.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling


def test_f2_kernels_keep_their_registers(enc_kernels):
    for k, regs in PARENT_REGS.items():
        assert enc_kernels[k]["regs"] <= regs, "%s: %d registers, %d before" % (k, enc_kernels[k]["regs"], regs)
