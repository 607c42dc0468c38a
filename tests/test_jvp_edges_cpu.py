"""The C restatement of finite_difference_jvp! (oracle/fd_oracle.c, src/jvp.jl:238-274) against the line-by-line Python
transcription (_literal_reference.finite_difference_jvp), bit for bit, before the device is held to it.

Compared: eps, every point f is called with (in order), the f-call count, jvp and the end state of cache.x1.  On
exact-dot inputs (_util.exact_dot_xv: dot(x, v) is exact in any summation order) eps is compared as each side computes
it; where an IEEE edge makes the dot inexact, the transcription's eps is fed to the oracle.  Covered: relstep / absstep
overrides (signed zeros, negative, subnormal), dir = +-1 and 0.3, edges in x and in v at indices 0, 31, 32, 33 and n-1,
negative and exactly-zero dots, f_in, cache.x1 aliased to x (JVPCache(x, fx1)), m != n, and hand-derived answers the two
restatements cannot share a wrong one on."""
import math

import numpy as np
import pytest

import _literal_reference as lit
from _util import GatherF, assert_same_bits, exact_dot_xv

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")

FD = {"forward": 0, "central": 1}
RELSTEPS = [None, 0.0, 1e-3, -1e-3, -0.0, 1.0]
ABSSTEPS = [None, 0.0, -0.0, 1e-160, 5e-324]
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 1e300, -1e300]
EXACT_EDGES = {0.0, np.inf, -np.inf}          # (and NaN): the dot stays order-independent with these in x or v


def _both(x, v, m, fdtype, *, f_in=False, alias=False, seed=0, feed=False, **kw):
    """Run the transcription and the oracle on the same GatherF; return (lit result, oracle result, lit points, oracle
    points, lit jvp, lit x1).  feed=True gives the oracle the transcription's eps."""
    n = x.size
    g = GatherF(m, n, seed)
    fin = None
    if f_in:
        fin = np.zeros(m)
        g.np_f([])(fin, x.copy())
    llog, olog = [], []
    xl = x.copy()
    cache = dict(x1=xl if alias else np.full(n, np.nan), fx1=np.full(m, np.nan))
    out = np.full(m, np.nan)
    with np.errstate(all="ignore"):
        rl = lit.finite_difference_jvp(out, g.np_f(llog), xl, v.copy(), cache, None if fin is None else fin.copy(),
                                       fdtype=fdtype, **kw)
    ro = oracle_mod().jvp(g.np_f(olog), x.copy(), v.copy(), m, fdtype=FD[fdtype], f_in=fin, alias_x1=alias,
                          eps_override=rl["eps"] if feed else None, **kw)
    return rl, ro, llog, olog, out, cache["x1"]


def oracle_mod():
    from oracle import fd_oracle
    return fd_oracle


def _check(rl, ro, llog, olog, out, x1, n, what, eps_bits=True):
    if eps_bits:
        assert_same_bits(np.array([ro["eps"]]), np.array([rl["eps"]]), f"{what}: eps")
    assert ro["fcalls"] == rl["fcalls"] == len(llog) == len(olog), what
    for i, (a, b) in enumerate(zip(olog, llog)):
        assert_same_bits(a, b, f"{what}: argument of f call {i}")
    assert_same_bits(ro["jvp"], out, f"{what}: jvp")
    assert_same_bits(ro["x1"][:n], x1, f"{what}: cache.x1")


@pytest.fixture(scope="module", autouse=True)
def _built(oracle):
    return oracle


def test_exact_dot_inputs_are_exact():
    from fractions import Fraction
    for kind in ("unit", "big", "tiny", "neg", "zero"):
        for n in (1, 33, 2049):
            x, v = exact_dot_xv(n, n, kind)
            exact = sum(Fraction(float(a)) * Fraction(float(b)) for a, b in zip(x, v))
            seq = 0.0
            for a, b in zip(x[::-1], v[::-1]):
                seq += float(a) * float(b)
            assert Fraction(float(np.dot(x, v))) == Fraction(seq) == exact, (kind, n)
            if kind == "neg":
                assert exact < 0
            if kind == "zero" and n % 2 == 0:
                assert exact == 0


# ------------------------------------------------------------------------------------------------ step overrides, dir
@pytest.mark.parametrize("absstep", ABSSTEPS)
@pytest.mark.parametrize("relstep", RELSTEPS)
@pytest.mark.parametrize("fdtype,dir", [("forward", 1.0), ("forward", -1.0), ("forward", 0.3), ("central", 1.0),
                                        ("central", -1.0)])
def test_oracle_matches_transcription_steps(fdtype, dir, relstep, absstep):
    for kind in ("unit", "tiny", "neg", "zero"):
        for n, m, f_in in ((40, 40, False), (37, 111, fdtype == "forward"), (2, 1, False)):
            x, v = exact_dot_xv(n, n + m, kind)
            r = _both(x, v, m, fdtype, f_in=f_in, relstep=relstep, absstep=absstep, dir=dir, seed=n)
            _check(*r, n, f"{kind} n={n} m={m} f_in={f_in}")


def test_central_ignores_dir():
    # epsilons.jl:50-53: the central step has no dir; dir = -1 and 0.3 give dir = 1's eps, points and jvp
    x, v = exact_dot_xv(64, 3, "neg")
    base = _both(x, v, 64, "central")
    for d in (-1.0, 0.3):
        r = _both(x, v, 64, "central", dir=d)
        assert_same_bits(np.array([r[1]["eps"]]), np.array([base[1]["eps"]]), f"dir={d}")
        assert r[1]["eps"] > 0
        assert_same_bits(r[1]["jvp"], base[1]["jvp"], f"dir={d}")
        for a, b in zip(r[3], base[3]):
            assert_same_bits(a, b, f"dir={d}: points")


# ------------------------------------------------------------------------------------------------ IEEE edges
@pytest.mark.parametrize("fdtype", list(FD))
@pytest.mark.parametrize("which", ["x", "v"])
@pytest.mark.parametrize("edge", EDGES)
def test_oracle_matches_transcription_edges(fdtype, which, edge):
    n = 64
    for kind in ("unit", "neg"):
        x, v = exact_dot_xv(n, 11, kind)
        for i in (0, 31, 32, 33, n - 1):
            (x if which == "x" else v)[i] = edge
        exact = np.isnan(edge) or edge in EXACT_EDGES or (edge == 0.0)
        r = _both(x, v, n, fdtype, feed=not exact, seed=5)
        _check(*r, n, f"{kind}: {edge!r} in {which}")
        if exact:                           # the oracle's own eps, no feeding
            r2 = _both(x, v, n, fdtype, seed=5)
            _check(*r2, n, f"{kind}: {edge!r} in {which} (own eps)")
            if np.isnan(edge) or (np.isinf(edge) and which == "x" and kind == "unit"):
                assert not np.isfinite(r2[1]["eps"])


@pytest.mark.parametrize("fdtype", list(FD))
def test_signed_zero_and_nan_v(fdtype):
    n = 70
    x, _ = exact_dot_xv(n, 9, "unit")
    vz = np.where(np.arange(n) % 3 == 0, -0.0, 0.0)                   # all-zero v, signed zeros mixed: dot = +-0
    r = _both(x, vz, n, fdtype, relstep=1e-3, absstep=2.0 ** -30)
    _check(*r, n, "zero v")
    assert r[1]["eps"] == 2.0 ** -30
    vn = np.full(n, np.nan)
    r = _both(x, vn, n, fdtype)
    _check(*r, n, "NaN v")
    assert np.isnan(r[1]["eps"]) and np.isnan(r[1]["jvp"]).all()


# ------------------------------------------------------------------------------------------------ aliasing
@pytest.mark.parametrize("fdtype", list(FD))
@pytest.mark.parametrize("kind", ["unit", "big", "neg"])
def test_aliased_x1(fdtype, kind):
    # JVPCache(x, fx1) keeps x1 === x (jvp.jl:73-80): central evaluates f at (x - eps v) + eps v; x ends as x1's end state
    n = 300
    x, v = exact_dot_xv(n, 21, kind)
    rl, ro, llog, olog, out, x1 = _both(x, v, n, fdtype, alias=True)
    _check(rl, ro, llog, olog, out, x1, n, "aliased")
    e = ro["eps"]
    if fdtype == "central":
        assert_same_bits(olog[0], x - e * v, "first point")
        assert_same_bits(olog[1], (x - e * v) + e * v, "second point: from the drifted x")
        assert_same_bits(ro["x1"][:n], (x - e * v) + e * v, "x's end state")
    else:
        assert_same_bits(olog[1], x + e * v)
        assert_same_bits(ro["x1"][:n], x + e * v)
    plain = _both(x, v, n, fdtype)
    assert_same_bits(np.array([plain[1]["eps"]]), np.array([e]))


# ------------------------------------------------------------------------------------------------ hand-derived answers
def test_hand_negative_zero_steps():
    # relstep = absstep = -0.0: eps = max(-0.0 * sqrt|d|, -0.0) * 1 = -0.0.  x + (-0.0) v keeps x_j except a -0.0 with
    # v_j < 0 or v_j = -0.0 (-0.0 * v_j = +0.0, and -0.0 + 0.0 = +0.0).  With f = 1/x, jvp_j = (1/x1_j - 1/x_j) / -0.0:
    # NaN where the point is unchanged, -Inf where -0.0 turned into +0.0 (Inf - (-Inf) = Inf, / -0.0 = -Inf).
    x = np.array([1.5, -0.0, -0.0, 0.0, 2.0, -0.0])
    v = np.array([1.0, -1.0, 1.0, -1.0, 0.5, -0.0])
    olog = []

    def inv(fx, xx):
        olog.append(xx.copy())
        with np.errstate(all="ignore"):
            fx[:] = 1.0 / xx

    r = oracle_mod().jvp(inv, x, v, 6, relstep=-0.0, absstep=-0.0)
    assert math.copysign(1.0, r["eps"]) == -1.0 and r["eps"] == 0.0
    assert_same_bits(olog[1], np.array([1.5, 0.0, -0.0, 0.0, 2.0, 0.0]), "x + eps v")
    assert_same_bits(r["jvp"], np.array([np.nan, -np.inf, np.nan, np.nan, np.nan, -np.inf]), "jvp")
    out, cache = np.zeros(6), dict(x1=np.zeros(6), fx1=np.zeros(6))
    with np.errstate(all="ignore"):
        rl = lit.finite_difference_jvp(out, lambda fx, xx: fx.__setitem__(slice(None), 1.0 / xx), x, v, cache,
                                       relstep=-0.0, absstep=-0.0)
    assert_same_bits(np.array([rl["eps"]]), np.array([-0.0]))
    assert_same_bits(out, r["jvp"])
    # central: -0.0 as well (no dir); x - (-0.0) v flips the other signs
    r = oracle_mod().jvp(inv, x, v, 6, fdtype=1, relstep=-0.0, absstep=-0.0)
    assert_same_bits(np.array([r["eps"]]), np.array([-0.0]))
    assert_same_bits(olog[2], np.array([1.5, -0.0, 0.0, 0.0, 2.0, -0.0]), "x - eps v")


def test_hand_nan_in_v():
    x, v = exact_dot_xv(40, 1, "unit")
    v[17] = np.nan
    for fd in (0, 1):
        log = []
        r = oracle_mod().jvp(lambda fx, xx: (log.append(xx.copy()), fx.__setitem__(slice(None), xx)), x, v, 40,
                             fdtype=fd)
        assert np.isnan(r["eps"]) and np.isnan(log[-1]).all() and np.isnan(r["jvp"]).all()


def test_hand_central_negative_dir_and_exact_eps():
    # eps = relstep * sqrt(|d|) with d exact; central ignores dir = -1: the step is positive, the points are x -+ eps v
    x = np.array([3.0, -1.0, 0.5, 2.0])
    v = np.array([-4.0, 2.0, 8.0, -0.25])                 # d = -12 - 2 + 4 - 0.5 = -10.5
    rel = 2.0 ** -20
    log = []
    r = oracle_mod().jvp(lambda fx, xx: (log.append(xx.copy()), fx.__setitem__(slice(None), xx * xx)), x, v, 4,
                         fdtype=1, relstep=rel, absstep=0.0, dir=-1.0)
    assert r["eps"] == rel * math.sqrt(10.5) > 0
    e = r["eps"]
    assert_same_bits(log[0], x - e * v)
    assert_same_bits(log[1], x + e * v)
    # exactly-zero dot: sqrt(0) = 0, so eps = absstep (forward: times dir)
    xz, vz = np.array([1.0, 1.0]), np.array([3.0, -3.0])
    assert oracle_mod().jvp(lambda fx, xx: None, xz, vz, 2, relstep=1e-3, absstep=1e-7, dir=-1.0)["eps"] == -1e-7
    assert oracle_mod().jvp(lambda fx, xx: None, xz, vz, 2, fdtype=1, relstep=1e-3, absstep=1e-7, dir=-1.0)["eps"] == 1e-7


def test_forward_f_in_skips_f_of_x():
    x, v = exact_dot_xv(50, 4, "unit")
    rl, ro, llog, olog, out, x1 = _both(x, v, 20, "forward", f_in=True)
    _check(rl, ro, llog, olog, out, x1, 50, "f_in")
    assert ro["fcalls"] == 1 and len(olog) == 1
    assert_same_bits(olog[0], x + ro["eps"] * v)
