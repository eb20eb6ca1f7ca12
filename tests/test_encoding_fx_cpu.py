"""The deterministic (64-bit fixed-point) lattice-gradient kernels of the permutohedral encoding, without a GPU.

A compile check of csrc/encoding.cu with the command `build()` uses: the fixed-point backward k_fx_enc_backward<D, F, POS> and double
backward k_fx_enc_double_backward<D, F, GOUT> exist for all 20 (D, F) pairs and both flag values, none of them spills, and the float
k_enc_* kernels are exactly the set the library had before them (their names, and so their template parameters, are unchanged)."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
PAIRS = [(D, F) for D in range(2, 7) for F in (1, 2, 4, 8)]


@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("encoding.cu",))}


def test_every_fixed_point_instantiation_is_built(kernels):
    expect = set()
    for D, F in PAIRS:
        for flag in ("false", "true"):
            expect.add("k_fx_enc_backward<%d, %d, %s>" % (D, F, flag))
            expect.add("k_fx_enc_double_backward<%d, %d, %s>" % (D, F, flag))
    assert {k for k in kernels if k.startswith("k_fx_enc_")} == expect
    assert "k_fx_flush" in kernels


def test_no_fixed_point_instantiation_spills(kernels):
    fx = {k: r for k, r in kernels.items() if k.startswith("k_fx_enc_")}
    assert len(fx) == 80
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in fx.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling


def test_float_kernels_are_the_same_set(kernels):
    expect = set()
    for D, F in PAIRS:
        expect.add("k_enc_forward<%d, %d>" % (D, F))
        for flags in ("false, true", "true, false", "true, true"):
            expect.add("k_enc_backward<%d, %d, %s>" % (D, F, flags))
            expect.add("k_enc_double_backward<%d, %d, %s>" % (D, F, flags))
    assert {k for k in kernels if k.startswith("k_enc_")} == expect
