"""IEEE edge inputs and overridden step sizes for the scalar paths (Hessian, gradient), CPU side.

fdbs_guarded's CPU twin (scalar_oracle/synth_scalar.c:synth_guarded) is pinned to an independent numpy evaluation in the
same blocked order at edge inputs; then the C restatements of hessians.jl:202-292 and gradients.jl:390-457, running the
native twin, are compared bit for bit with the line-by-line Python transcriptions (tests/_util.py) on edge x, with every
relstep / absstep the GPU file uses, negative relstep included: every point f sees, H or df, and f(x)."""
import itertools

import numpy as np
import pytest

from _util import assert_same_bits, gradient_transcribed, guarded_numpy, hessian_transcribed, max_julia
from scalar_oracle import fd_scalar_oracle as so

f64 = np.float64
EDGES = [0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1e-160, 1.0, -2.5]
RELSTEPS = [None, 0.0, 1e-3, 1e-12, -1e-3]
ABSSTEPS = [None, 0.0, 1e-6, 1e-160, 1e-320, 5e-324]


@pytest.fixture(scope="module")
def soracle():
    so.build()
    so.lib()
    return so


def _coeffs(n, seed):
    rng = np.random.default_rng(seed + n)
    return 0.5 + rng.random(n), rng.random(n) * 2 - 1


def _edge_x(rng, n, p=0.4):
    """ordinary values of both signs and magnitudes, each component replaced by an edge value with probability p"""
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
    for k in range(n):
        if rng.random() < p:
            x[k] = EDGES[rng.integers(len(EDGES))]
    return x


# ------------------------------------------------------------------------------------------------ the test function
@pytest.mark.parametrize("n", [1, 31, 33, 1025])
def test_synth_guarded_matches_numpy(soracle, n):
    a, w = _coeffs(n, 3)
    twin = so.SynthScalar(n, a, w, name="synth_guarded")
    rng = np.random.default_rng(500 + n)
    xs = [_edge_x(rng, n, p) for p in (0.0, 0.1, 0.5, 1.0) for _ in range(4)]
    xs += [np.full(n, v) for v in EDGES]                                  # every component the same edge value
    for t, x in enumerate(xs):
        got = twin(x)
        ref = guarded_numpy(x, a, w)
        assert np.isfinite(got), f"n={n} x #{t}: f is not finite"
        assert_same_bits(np.array([got]), np.array([ref]), f"n={n} x #{t}")


def test_synth_guarded_sees_zero_signs_not_nan_signs(soracle):
    # the two properties the edge tests rely on, checked on the C twin: f(-0.0 at k) - f(+0.0 at k) carries w_k,
    # and the sign and payload of a NaN change nothing
    n = 40
    a, w = _coeffs(n, 3)
    twin = so.SynthScalar(n, a, w, name="synth_guarded")
    x = np.random.default_rng(8).standard_normal(n)
    for k in (0, 31, 32, n - 1):
        xp, xm = x.copy(), x.copy()
        xp[k], xm[k] = 0.0, -0.0
        assert twin(xp) != twin(xm)
        nans = [np.float64(np.nan), -np.float64(np.nan), np.frombuffer(np.uint64(0x7FF0000000000001).tobytes(), f64)[0],
                np.frombuffer(np.uint64(0xFFF8DEADBEEF0000).tobytes(), f64)[0]]
        vals = []
        for v in nans:
            xn = x.copy()
            xn[k] = v
            vals.append(twin(xn))
        assert all(np.isfinite(vals)) and len({f64(v).tobytes() for v in vals}) == 1


# ------------------------------------------------------------------------------------------------ restatement vs transcription
def _hessian_case(soracle, n, x, relstep, absstep, what):
    a, w = _coeffs(n, 5)
    twin = so.SynthScalar(n, a, w, name="synth_guarded")
    H, fx, pts = hessian_transcribed(lambda v: guarded_numpy(v, a, w), x, relstep, absstep)
    r = soracle.hessian(twin.native("synth_guarded"), x, relstep=relstep, absstep=absstep, log=True)
    assert r["fcalls"] == len(pts) == 2 * n * n + 1, what
    for k, (p, q) in enumerate(zip(r["points"], pts)):
        assert_same_bits(p, q, f"{what}: point {k}")
    assert_same_bits(r["H"][:n, :n], H, f"{what}: H")
    assert_same_bits(np.array([r["fx"]]), np.array([fx]), f"{what}: fx")
    assert np.isfinite(fx)


def _step_sizes(x, relstep, absstep):
    relstep = f64(2.0 ** -13) if relstep is None else f64(relstep)
    absstep = relstep if absstep is None else f64(absstep)
    with np.errstate(all="ignore"):
        return np.array([max_julia(relstep * abs(v), absstep) for v in x])


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_hessian_oracle_matches_transcription_edges(soracle, n):
    rng = np.random.default_rng(202 + n)
    for relstep, absstep in itertools.product(RELSTEPS, ABSSTEPS):
        x = _edge_x(rng, n)
        _hessian_case(soracle, n, x, relstep, absstep, f"n={n} relstep={relstep} absstep={absstep} x={x}")


def test_hessian_transcription_reaches_step_edges(soracle):
    # the three step-size edges of the GPU file, fed to both restatements and checked to be reached:
    #   eps = 0 on a +-0.0 component; eps_i * eps_j subnormal or flushed to 0 while (4 eps_i) * eps_j is not (the
    #   operation order of the off-diagonal denominator matters); eps_i * eps_i overflowing (1e300, default step)
    x = np.array([-0.0, 1.0, 0.0, 1e300, -2.5, 1e-320, 7.0, 5e-324])
    n = x.size
    cases = {"zero eps": (None, 0.0), "subnormal product": (None, 1e-320), "absstep 1e-160": (1e-3, 1e-160),
             "overflow": (None, None), "negative relstep": (-1e-3, None)}
    for name, (rel, ab) in cases.items():
        e = _step_sizes(x, rel, ab)
        with np.errstate(all="ignore"):
            if name == "zero eps":
                assert e[0] == 0 and e[2] == 0
            if name.startswith("subnormal"):
                p4, q4 = (f64(4) * e[:, None]) * e[None, :], f64(4) * (e[:, None] * e[None, :])
                assert np.any(p4.view(np.uint64) != q4.view(np.uint64)), name
            if name == "overflow":
                assert np.isinf(e[3] * e[3]) and np.isfinite(e[3])
            if name == "negative relstep":
                assert np.all(np.signbit(e[np.isfinite(e)]))
        _hessian_case(soracle, n, x, rel, ab, name)


@pytest.mark.parametrize("n", [1, 2, 5, 8])
def test_gradient_oracle_matches_transcription_edges(soracle, n):
    a, w = _coeffs(n, 7)
    twin = so.SynthScalar(n, a, w, name="synth_guarded")
    f_py = lambda v: guarded_numpy(v, a, w)
    rng = np.random.default_rng(390 + n)
    for relstep, absstep in itertools.product(RELSTEPS, ABSSTEPS):
        for fd, fx, dir in ((0, None, 1.0), (0, "f(x)", 1.0), (0, None, -1.0), (1, None, 1.0)):
            x = _edge_x(rng, n)
            fxv = twin(x) if fx else None
            what = f"n={n} fdtype={fd} fx={fxv} dir={dir} relstep={relstep} absstep={absstep} x={x}"
            df, pts = gradient_transcribed(f_py, x, fd, fxv, relstep, absstep, dir)
            r = soracle.gradient(twin.native("synth_guarded"), x, fd, fx=fxv, relstep=relstep, absstep=absstep, dir=dir,
                                 log=True)
            assert r["fcalls"] == len(pts) == (2 * n if fd == 1 else n + (fxv is None)), what
            for k, (p, q) in enumerate(zip(r["points"], pts)):
                assert_same_bits(p, q, f"{what}: point {k}")
            assert_same_bits(r["df"], df, f"{what}: df")
