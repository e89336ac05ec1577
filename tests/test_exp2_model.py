"""CPU (-m "not gpu"): numpy model of the table-based exp2 the TMA-staged SEIso Gram / trace kernels use
(csrc/gram_fast.cu: exp2_tab + seiso_fast_prepare).  The model re-executes the kernel's steps -- magic-number rounding, 64-entry
table, degree-5 polynomial whose coefficients are READ FROM THE SOURCE, exponent added in the integer pipe, integer underflow
guard -- in IEEE double without fma, so it bounds the algorithm's error rather than reproducing the device bits.  The model
that does reproduce them, with an exact fma, is tests/seiso_model.py (tested against this one in tests/test_seiso_model.py);
the device kernels are compared with it bit for bit in tests/test_gpu_seiso_kernel_contracts.py and with the oracle in
tests/test_gpu_parity.py.  What the reference computes here is
exp(-r^2 / (2 l^2)) * sigma^2 (src/kernels/se_iso.jl:27, cov(se, r) = σ² exp(-r/(2ℓ²)) over the squared distance)."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT

SRC = open(os.path.join(ROOT, "gaussianprocesses.jl_b200", "csrc", "gram_fast.cu")).read()


def _coeffs():
    body = SRC[SRC.index("double exp2_tab("):]
    body = body[:body.index("return ((unsigned)")]
    lead = float(re.search(r"double p = ([0-9.eE+-]+);", body).group(1))
    rest = [float(m) for m in re.findall(r"p = fma\(p, f, ([0-9.eE+-]+)\);", body)]
    return [lead] + rest


def _prepare(l2, s2):
    """seiso_fast_prepare: c = -log2(e) / (2 l^2) in long double, table s2 * 2^(j/64)."""
    c = np.longdouble(-0.5) / np.longdouble(l2) * np.longdouble("1.442695040888963407359924681001892137")
    tab = (np.longdouble(s2) * np.exp2(np.arange(64, dtype=np.longdouble) / np.longdouble(64))).astype(np.float64)
    return float(c), tab


def _exp2_tab(z, tab, co):
    z = np.asarray(z, dtype=np.float64)
    MAGIC = 6755399441055744.0
    zs = z * 64.0 + MAGIC
    ki = (zs.view(np.int64) & 0xFFFFFFFF).astype(np.uint32).view(np.int32).astype(np.int64)      # __double2loint
    kf = zs - MAGIC
    f = z - kf * 0.015625
    p = np.full_like(z, co[0])
    for c in co[1:]:
        p = p * f + c
    r = tab[ki & 63] * p
    bits = r.view(np.int64)
    hi = (bits >> 32) + ((ki >> 6) << 20)                                                        # exponent add on the high word
    v = ((hi << 32) | (bits & 0xFFFFFFFF)).view(np.float64)
    zhi = (z.view(np.int64) >> 32) & 0xFFFFFFFF
    return np.where(zhi > 0xC08E0000, 0.0, v), f


def test_polynomial_is_the_taylor_series_of_exp2():
    co = _coeffs()
    assert len(co) == 6
    ln2 = np.log(2.0)
    want = [ln2 ** 5 / 120, ln2 ** 4 / 24, ln2 ** 3 / 6, ln2 ** 2 / 2, ln2, 1.0]
    assert np.allclose(co, want, rtol=4e-16, atol=0)


@pytest.mark.parametrize("s2", [1e-15 * 1.0001, 0.37, 1.0, np.exp(0.6), 9.9e14])
def test_exp2_table_model_accuracy_and_range(s2):
    co = _coeffs()
    _, tab = _prepare(1.0, s2)
    rng = np.random.default_rng(3)
    z = -np.concatenate([rng.uniform(0, 1, 20000), rng.uniform(0, 60, 40000), rng.uniform(60, 959.9, 20000),
                         np.arange(0, 961) / 1.0, np.arange(0, 4096) / 64.0, [0.0, 1e-300, 1e-17, 959.999999]])
    v, f = _exp2_tab(z, tab, co)
    assert np.max(np.abs(f)) <= 1.0 / 128 + 1e-18                     # the reduced argument stays inside the fit interval
    want = (np.longdouble(s2) * np.exp2(z.astype(np.longdouble)))
    rel = np.abs((v.astype(np.longdouble) - want) / want).astype(np.float64)
    assert np.all(np.isfinite(v)) and np.all(v > 0)
    assert rel.max() < 4.5e-16, rel.max()                             # < 2 ulp: table rounding + product + polynomial tail 3.5e-17
    # exact points: z = -k/64 with a representable table entry returns the table entry scaled by a power of two
    zz = -np.arange(0, 2048) / 64.0
    vv, _ = _exp2_tab(zz, tab, co)
    assert np.array_equal(vv, np.ldexp(tab[(-np.arange(0, 2048)) & 63], -((np.arange(0, 2048) + 63) // 64)))
    # underflow guard (high-word compare, granularity 2^-11 at this magnitude): below -960.0005 the result is a clean zero
    # (the exponent add would wrap), never garbage; between -960 and there it is still the correct normal number
    zu = -np.concatenate([[960.0005, 1000.0, 1074.0, 5e4, 1e9, 1e300], rng.uniform(960.01, 4e6, 2000)])
    vu, _ = _exp2_tab(zu, tab, co)
    assert np.all(vu == 0.0)
    # just above the guard the value is still a normal number for every admissible s2 (1e-15 .. 1e15)
    ve, _ = _exp2_tab(np.array([-960.0, -959.5]), tab, co)
    assert np.all(ve >= np.finfo(np.float64).tiny)


def test_gram_value_error_budget_at_the_contract_sizes():
    """Whole-entry error budget of exp2_tab(r2 * c_hi): rounding c to double shifts z by |z| 2^-53, i.e. a relative error
    |z| ln2 2^-53 in k; entries below 1e-18 sigma^2 (|z| > 60) carry < 5e-15 relative error -- 4 orders inside the 1e-10 gate."""
    co = _coeffs()
    rng = np.random.default_rng(5)
    for ll, lsig in ((0.3, 0.3), (-1.0, 0.7), (1.5, -2.0)):
        l2, s2 = np.exp(2 * ll), np.exp(2 * lsig)
        c, tab = _prepare(l2, s2)
        r2 = rng.uniform(0, 120 * l2, 50000)
        v, _ = _exp2_tab(r2 * c, tab, co)
        want = np.longdouble(s2) * np.exp(-np.longdouble(0.5) * r2.astype(np.longdouble) / np.longdouble(l2))
        rel = np.abs((v.astype(np.longdouble) - want) / want).astype(np.float64)
        assert rel.max() < 2e-14, rel.max()
