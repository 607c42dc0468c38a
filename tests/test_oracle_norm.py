"""Pins the one piece of third-party arithmetic on the hot path — LinearAlgebra.norm at jacobians.jl:560,601, i.e.
OpenBLAS dnrm2 for vectors of 32 or more elements — against OpenBLAS itself.

  * golden: oracle.norm2 reproduces, BIT FOR BIT, the values OpenBLAS's dnrm2 binary returned for the deterministic
    vectors of tests/golden/dnrm2_vectors.py (tests/golden/dnrm2_openblas.json, made by make_dnrm2_golden.py) — sizes
    32 .. 10^7, the masked vectors x .* (colorvec .== k) of the benchmark colourings, magnitudes 1e-200 .. 1e200;
  * live: where scipy's BLAS is importable, the same on fresh random vectors;
  * the n < 32 branch (stdlib generic_norm2) against its definition: in-order Float64 sum, scaling only when needed;
  * the step size the driver derives from it (jacobians.jl:559-561) uses exactly this norm.
"""
import json
import sys
from pathlib import Path

import numpy as np
import pytest

GOLD = Path(__file__).resolve().parent / "golden"
sys.path.insert(0, str(GOLD))
from dnrm2_vectors import vector  # noqa: E402


def _cases():
    return json.loads((GOLD / "dnrm2_openblas.json").read_text())["cases"]


@pytest.mark.parametrize("case", _cases(), ids=lambda c: f"{c['kind']}-n{c['n']}-e{c['scale_exp']}")
def test_norm_matches_openblas_dnrm2_golden(oracle, case):
    x = vector(case["seed"], case["n"], case["kind"], case["scale_exp"])
    assert oracle.norm2(x).hex() == case["dnrm2_hex"]


def test_golden_shows_what_a_plain_sum_would_miss():
    # the fixture is not vacuous: at the benchmark's size the in-order Float64 sum is tens to hundreds of ulps away
    big = [c for c in _cases() if c["n"] >= 1_000_000 and c["plain_double_sum_ulps"] is not None]
    assert big and max(abs(c["plain_double_sum_ulps"]) for c in big) > 50


def test_norm_matches_openblas_dnrm2_live(oracle):
    blas = pytest.importorskip("scipy.linalg.blas")
    # OpenBLAS picks its kernels per CPU at run time: only a host whose dnrm2 is the x87 kernel the fixture was recorded
    # from can serve as a live reference (every x86-64 target known to us uses it; anything else is skipped, not failed)
    probe = [c for c in _cases() if c["n"] <= 100003][:12]
    if any(float(blas.dnrm2(vector(c["seed"], c["n"], c["kind"], c["scale_exp"]))).hex() != c["dnrm2_hex"] for c in probe):
        pytest.skip("this host's OpenBLAS dnrm2 is not the kernel tests/golden/dnrm2_openblas.json was recorded from")
    rng = np.random.default_rng(77)
    for t in range(120):
        n = int(rng.integers(32, 300_000))
        x = rng.normal(size=n) * 10.0 ** rng.uniform(-6, 6)
        if t % 3 == 0:
            x[rng.random(n) < 0.66] = 0.0
        assert oracle.norm2(x) == float(blas.dnrm2(x)), (t, n)


def test_generic_norm2_below_32_elements(oracle):
    rng = np.random.default_rng(5)
    for n in range(1, 32):
        x = rng.normal(size=n)
        s = 0.0
        for v in x:                      # in-order Float64 accumulation, then sqrt (stdlib generic_norm2, unscaled branch)
            s += v * v
        assert oracle.norm2(x) == float(np.sqrt(s))
    assert oracle.norm2(np.zeros(7)) == 0.0 and oracle.norm2(np.array([])) == 0.0
    assert oracle.norm2(np.array([3.0, -4.0])) == 5.0
    assert oracle.norm2(np.array([1.0, np.inf])) == np.inf
    # scaled branch: the squares would overflow / underflow
    big = np.full(5, 1e200)
    assert oracle.norm2(big) == 1e200 * float(np.sqrt(5.0))
    tiny = np.full(5, 1e-200)
    assert oracle.norm2(tiny) == 1e-200 * float(np.sqrt(5.0))


def _in_order_norm(x):
    s = 0.0
    for v in x:
        s += float(v) * float(v)
    return float(np.sqrt(s))


def _scaled_norm(x):
    m = float(np.max(np.abs(x)))
    s = 0.0
    for v in x:
        t = abs(float(v)) / m
        s += t * t
    return m * float(np.sqrt(s))


@pytest.mark.parametrize("n", [13, 31])
def test_generic_norm2_branches_at_the_ends_of_the_range(oracle, n):
    # generic_norm2 scales only when maxabs^2 == 0 or n*maxabs^2 overflows; otherwise it keeps the in-order Float64 sum,
    # however lossy (the device step-size pass follows the same rule for n < 32)
    rng = np.random.default_rng(n)
    sub = rng.uniform(0.5, 1.5, n) * 1e-160 * np.where(rng.random(n) < 0.5, -1.0, 1.0)   # squares subnormal, nonzero
    r = oracle.norm2(sub)
    assert r == _in_order_norm(sub)
    assert abs(r / _scaled_norm(sub) - 1) > 1e-9         # the lossy value, not the accurate one
    zero_sq = rng.uniform(0.5, 1.5, n) * 1e-170              # every square underflows to 0
    assert oracle.norm2(zero_sq) == _scaled_norm(zero_sq) and oracle.norm2(zero_sq) > 0
    big = rng.uniform(0.5, 1.5, n) * 1e150                    # n*maxabs^2 overflows, the sum of squares itself does not
    big[n // 3] = -1.2e154
    m = float(np.max(np.abs(big)))
    assert np.isinf(n * m * m) and np.isfinite(float(np.sum(big * big)))
    assert oracle.norm2(big) == _scaled_norm(big)
    huge = np.full(n, 1e300)                                  # squares overflow
    assert oracle.norm2(huge) == _scaled_norm(huge) == 1e300 * float(np.sqrt(float(n)))
    mixed = np.zeros(n)
    mixed[[0, n // 2]] = [5e-324, -0.0]                       # the smallest subnormal: its square is 0
    assert oracle.norm2(mixed) == 5e-324


def test_subnormal_square_sums_to_a_normal_number(oracle):
    # 10^5 equal components whose squares are subnormal and each rounded by nearly half an ulp: the plain Float64 sum is
    # a normal number but 1.07e-11 off; dnrm2 (x87 extended) is not
    from fractions import Fraction
    v = 4.79825341824841e-157
    sq = v * v
    err = abs(Fraction(sq) - Fraction(v) ** 2) / Fraction(5e-324)
    assert 0.45 < err <= 0.5
    x = np.full(100_000, v)
    r = oracle.norm2(x)
    assert r == 1.517340959235351e-154
    plain = float(np.sqrt(np.sum(x * x)))
    assert abs(plain / r - 1) > 5e-12


@pytest.mark.parametrize("fdtype", [0, 1])
def test_driver_step_size_uses_this_norm(oracle, fdtype):
    # the eps the oracle's colour loop reports == compute_epsilon(sqrt(norm(x .* (color .== k)))) with fdo_norm2
    n = 100
    rng = np.random.default_rng(9)
    x = 0.5 + rng.random(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    colptr = np.arange(1, n + 2, dtype=np.int64)
    rowval = np.arange(1, n + 1, dtype=np.int64)
    J = np.zeros(n)

    def f(fx, xx):
        fx[:] = xx * xx

    eps = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), J, f, x.copy(), fdtype=fdtype, colorvec=cv)["eps"]
    for k in (1, 2, 3):
        assert eps[k - 1] == oracle.color_eps(x, cv, k, fdtype)
