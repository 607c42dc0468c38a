"""The two CPU restatements of the reference's colour loop (the C oracle and the literal transcription,
tests/_literal_reference.py) on IEEE edge inputs: signed zeros in every colour, NaN and +-Inf components, a colour that is
all NaN or all zero, magnitudes from 1e-320 to 1e300, and a colour that mixes 1e200 with 1e-200.

Bars, bit for bit (tests/_util.assert_same_bits: bit patterns, every NaN one class): the step sizes, J, the end state of
cache.x1 and of the caller's x, and EVERY argument f! is called with.  The last one pins the signed-zero semantics of
the perturbed points: Julia's `Bool * Float64` is a strong zero (`false * v == copysign(0.0, v)`, never NaN), so
`x1 .+ eps .* (colour .== k)` adds a signed zero to every other component, and `max` propagates NaN.

The two restatements could still agree on a wrong answer, so a few known answers are derived by hand below."""
import numpy as np
import pytest
import scipy.sparse as sps

import _literal_reference as lit
from _util import assert_same_bits, cyc_colors, f_tridiag, tridiag_csc

# NaN and Inf are the data here: numpy's warnings about producing them are expected
pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")

FD = {"forward": 0, "central": 1}
KINDS = ["csc_same", "csc_to_dense", "proto_to_dense", "banded", "banded_to_dense", "dense_cols"]


def _setup(kind, long_x, seed):
    rng = np.random.default_rng(seed)
    n = 40 if long_x else 13                     # 32 or more components: norm takes its BLAS (dnrm2) branch
    m = n + 1
    if kind in ("banded", "banded_to_dense"):
        l, u = 1, 2
        D = np.zeros((m, n), bool)
        for c in range(n):
            D[max(0, c - u):min(m, c + l + 1), c] = True
    else:
        l = u = 0
        D = rng.random((m, n)) < 0.3
        D[np.arange(min(m, n)), np.arange(min(m, n))] = True
    W = sps.csr_matrix(rng.uniform(-1, 1, (m, n)) * D)    # only the structural entries enter f: no 0 * Inf
    q = rng.integers(0, n, m)

    def f(fx, x):                                         # sign-sensitive: copysign sees the sign of a zero
        fx[:] = W @ x + 0.1 * x[q] ** 2 + np.copysign(0.5, x[q])

    if kind == "dense_cols":
        cv = np.arange(1, n + 1, dtype=np.int64)
    else:
        cv = cyc_colors(n, 3)
        if long_x:
            cv[-1] = 0                                    # a component no colour perturbs
    return dict(kind=kind, m=m, n=n, l=l, u=u, D=D, f=f, cv=cv, rng=rng)


def _edge_inputs(S):
    """name -> x.  'Colour 2' is the second colour (the second column for dense_cols)."""
    rng, n, cv = S["rng"], S["n"], S["cv"]
    base = rng.uniform(-2, 2, n)
    col = lambda k: np.flatnonzero(cv == k)           # noqa: E731
    out = {}
    x = base.copy()
    for k in range(1, int(cv.max()) + 1):
        idx = col(k)
        x[idx[0]] = -0.0
        if len(idx) > 1:
            x[idx[-1]] = 0.0
    out["signed_zeros"] = x
    x = base.copy(); x[col(2)[0]] = np.nan; out["nan"] = x                          # noqa: E702
    x = base.copy(); x[col(2)[0]] = np.inf; out["+inf"] = x                         # noqa: E702
    x = base.copy(); x[col(2)[0]] = -np.inf; out["-inf"] = x                        # noqa: E702
    x = base.copy(); x[col(2)[0]] = np.nan; x[col(2)[-1]] = np.inf; x[0] = -0.0; out["nan_inf"] = x  # noqa: E702
    x = base.copy(); x[col(2)] = np.nan; out["nan_colour"] = x                      # noqa: E702
    x = base.copy(); x[col(2)] = np.where(np.arange(len(col(2))) % 2, 0.0, -0.0); out["zero_colour"] = x  # noqa: E702
    out["magnitudes"] = np.copysign(10.0 ** rng.uniform(-320, 300, n), base)
    x = base.copy()
    x[col(2)] = np.copysign(np.where(np.arange(len(col(2))) % 2, 1e200, 1e-200), base[col(2)])
    out["mixed_colour"] = x
    return out


def _recording(f, log):
    def g(fx, x):
        log.append(np.array(x, copy=True))
        f(fx, x)
    return g


def _literal_target(S):
    kind, m, n, l, u, D = S["kind"], S["m"], S["n"], S["l"], S["u"], S["D"]
    A = sps.csc_matrix(D)
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    if kind == "csc_same":
        J = lit.CSC(m, n, colptr, rowval, np.full(A.nnz, np.nan)); sparsity = J                            # noqa: E702
        P = lambda o: o.Problem.csc_same(m, n, colptr, rowval)                                            # noqa: E731
    elif kind == "csc_to_dense":
        J = np.full((m, n), np.nan); sparsity = lit.CSC(m, n, colptr, rowval)                            # noqa: E702
        P = lambda o: o.Problem.csc_to_dense(m, n, colptr, rowval)                                        # noqa: E731
    elif kind == "proto_to_dense":
        J = np.full((m, n), np.nan); sparsity = D.astype(np.float64)                                      # noqa: E702
        P = lambda o: o.Problem.coo_to_dense(m, n, *o.findstructralnz_dense(D.astype(np.float64)))        # noqa: E731
    elif kind == "banded":
        J = lit.Banded(m, n, l, u, np.full((l + u + 1, n), np.nan)); sparsity = J                         # noqa: E702
        P = lambda o: o.Problem.banded(m, n, l, u)                                                        # noqa: E731
    elif kind == "banded_to_dense":
        J = np.full((m, n), np.nan); sparsity = lit.Banded(m, n, l, u)                                    # noqa: E702
        P = lambda o: o.Problem.banded_to_dense(m, n, l, u)                                               # noqa: E731
    else:
        J = np.full((m, n), np.nan); sparsity = None                                                      # noqa: E702
        P = lambda o: o.Problem.dense(m, n)                                                               # noqa: E731
    return J, sparsity, P


def _flat(J):
    if isinstance(J, lit.CSC):
        return J.nzval
    if isinstance(J, lit.Banded):
        return J.data.reshape(-1, order="F")
    return J.reshape(-1, order="F")


def _both(oracle, S, x, fdtype, dir, absstep):
    m, n, f, cv = S["m"], S["n"], S["f"], S["cv"]
    J, sparsity, P = _literal_target(S)
    kw = {} if absstep is None else {"absstep": absstep}
    log_l, log_o = [], []
    cache_l = dict(x1=np.full(n, np.nan), x2=np.full(n, np.nan), fx=np.full(m, np.nan), fx1=np.full(m, np.nan))
    xl = x.copy()
    rl = lit.finite_difference_jacobian(J, _recording(f, log_l), xl, cache_l, None, fdtype=fdtype, colorvec=cv,
                                        sparsity=sparsity, dir=dir, **kw)
    Jl = _flat(J)
    dense = S["kind"] == "dense_cols"
    Jo = np.full(Jl.size, np.nan)
    cache_o = dict(x1=np.full(n, np.nan), x2=np.full(n, np.nan), fx=np.full(m, np.nan), fx1=np.full(m, np.nan))
    xo = x.copy()
    ro = oracle.jacobian(P(oracle), Jo, _recording(f, log_o), xo, fdtype=FD[fdtype], colorvec=None if dense else cv,
                         dir=dir, cache=cache_o, **kw)
    return dict(rl=rl, ro=ro, Jl=Jl, Jo=Jo, xl=xl, xo=xo, cache_l=cache_l, cache_o=cache_o, log_l=log_l, log_o=log_o)


@pytest.mark.parametrize("absstep", [None, 0.0], ids=["absstep_default", "absstep_0"])
@pytest.mark.parametrize("dir", [1.0, -1.0], ids=["dir+", "dir-"])
@pytest.mark.parametrize("long_x", [False, True], ids=["n13", "n40"])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("kind", KINDS)
def test_edge_inputs_oracle_matches_literal(oracle, kind, fdtype, long_x, dir, absstep):
    S = _setup(kind, long_x, 4242 + 10 * KINDS.index(kind) + long_x)
    for name, x in _edge_inputs(S).items():
        what = f"{kind} {fdtype} n={S['n']} dir={dir} absstep={absstep} x={name}"
        r = _both(oracle, S, x, fdtype, dir, absstep)
        assert r["ro"]["fcalls"] == r["rl"]["fcalls"] == len(r["log_o"]) == len(r["log_l"]), what
        assert_same_bits(r["ro"]["eps"], r["rl"]["eps"], f"{what}: eps")
        for i, (a, b) in enumerate(zip(r["log_o"], r["log_l"])):
            assert_same_bits(a, b, f"{what}: argument of f! call {i}")
        assert_same_bits(r["Jo"], r["Jl"], f"{what}: J")
        assert_same_bits(r["cache_o"]["x1"], r["cache_l"]["x1"], f"{what}: cache.x1 end state")
        assert_same_bits(r["xo"], r["xl"], f"{what}: caller's x end state")


@pytest.mark.parametrize("long_x", [False, True], ids=["n13", "n40"])
@pytest.mark.parametrize("kind", KINDS)
def test_edge_inputs_complex_step_oracle_matches_literal(oracle, kind, long_x):
    S = _setup(kind, long_x, 5151 + 10 * KINDS.index(kind) + long_x)
    m, n, cv, D = S["m"], S["n"], S["cv"], S["D"]
    Wc = sps.csr_matrix(np.random.default_rng(9).uniform(-1, 1, (m, n)) * D)

    def f(fx, x):                       # linear in x, scaled by a factor that sees the sign of real(x[0]) when it is a zero
        fx[:] = (Wc @ x) * (1.0 + np.arctan2(0.0, x[0].real))

    for name, x in _edge_inputs(S).items():
        what = f"{kind} n={n} x={name}"
        J, sparsity, P = _literal_target(S)
        log_l, log_o = [], []
        cache = dict(x1=np.zeros(n, np.complex128), fx=np.zeros(m, np.complex128))
        rl = lit.finite_difference_jacobian_complex(J, _recording(f, log_l), x.copy(), cache, colorvec=cv, sparsity=sparsity)
        Jl = _flat(J)
        Jo = np.full(Jl.size, np.nan)
        ro = oracle.jacobian_complex(P(oracle), Jo, _recording(f, log_o), x.copy(),
                                     colorvec=None if kind == "dense_cols" else cv)
        assert ro["fcalls"] == rl["fcalls"] == len(log_o) == len(log_l), what
        for i, (a, b) in enumerate(zip(log_o, log_l)):
            assert_same_bits(a.view(np.float64), b.view(np.float64), f"{what}: argument of f! call {i}")
        assert_same_bits(Jo, Jl, f"{what}: J")


# ------------------------------------------------------------------------------------------- hand-derived known answers
# Tridiagonal n = 40, colours 1, 2, 3 cyclic, component 2 (0-based; colour 3) set to -0.0.  The other components are
# nonzero, so every colour's step is nonzero.
N40 = 40
J0 = 2


def _tridiag_x():
    x = np.random.default_rng(3).uniform(0.5, 2.0, N40)
    x[J0] = -0.0
    return x


def _tridiag_runs(oracle, fdtype, dir=1.0, absstep=None):
    """(oracle, literal) -> dict(args=[x seen by each f! call], eps=...)"""
    colptr, rowval = tridiag_csc(N40)
    cv = cyc_colors(N40, 3)
    kw = {} if absstep is None else {"absstep": absstep}
    out = []
    log = []
    r = oracle.jacobian(oracle.Problem.csc_same(N40, N40, colptr, rowval), np.zeros(len(rowval)), _recording(f_tridiag, log),
                        _tridiag_x(), fdtype=FD[fdtype], colorvec=cv, dir=dir, **kw)
    out.append(dict(args=log, eps=r["eps"]))
    log = []
    J = lit.CSC(N40, N40, colptr, rowval)
    cache = dict(x1=np.zeros(N40), x2=np.zeros(N40), fx=np.zeros(N40), fx1=np.zeros(N40))
    r = lit.finite_difference_jacobian(J, _recording(f_tridiag, log), _tridiag_x(), cache, None, fdtype=fdtype, colorvec=cv,
                                       sparsity=J, dir=dir, **kw)
    out.append(dict(args=log, eps=r["eps"]))
    return out


@pytest.mark.parametrize("dir,expect", [(1.0, [True, False, False, False]), (-1.0, [True, True, False, True])])
def test_kat_signed_zero_forward(oracle, dir, expect):
    # call 0 is f(x): the caller's -0.0.  Colour 1: x1 + eps1*false = -0.0 + copysign(0, eps1).  eps1 > 0 gives +0.0;
    # eps1 < 0 (dir = -1) gives -0.0 + -0.0 = -0.0.  Either way the restore x1 - copysign(0, eps1) leaves +0.0
    # (+0.0 - +0.0 and -0.0 - -0.0 are both +0.0), so colour 2 sees +0.0 + (+-0.0) = +0.0.  Colour 3 perturbs the
    # component itself: +0.0 + eps3, which is eps3 and has the sign of dir.
    for r in _tridiag_runs(oracle, "forward", dir):
        assert [bool(np.signbit(a[J0])) for a in r["args"]] == expect
        assert r["args"][3][J0] == r["eps"][2]


def test_kat_signed_zero_forward_zero_step(oracle):
    # absstep = 0 and dir = -1 with colour 3 all zero: eps3 = max(0*relstep, 0) * -1 = -0.0.  The component keeps +0.0
    # from colour 1 on (see above), and at colour 3 it is +0.0 + -0.0 = +0.0, not the caller's -0.0.
    colptr, rowval = tridiag_csc(N40)
    cv = cyc_colors(N40, 3)
    for runner in ("oracle", "literal"):
        x = _tridiag_x()
        x[cv == 3] = -0.0
        log = []
        if runner == "oracle":
            r = oracle.jacobian(oracle.Problem.csc_same(N40, N40, colptr, rowval), np.zeros(len(rowval)),
                                _recording(f_tridiag, log), x, fdtype=0, colorvec=cv, dir=-1.0, absstep=0.0)
        else:
            J = lit.CSC(N40, N40, colptr, rowval)
            cache = dict(x1=np.zeros(N40), x2=np.zeros(N40), fx=np.zeros(N40), fx1=np.zeros(N40))
            r = lit.finite_difference_jacobian(J, _recording(f_tridiag, log), x, cache, None, colorvec=cv, sparsity=J,
                                               dir=-1.0, absstep=0.0)
        assert np.signbit(r["eps"][2]) and r["eps"][2] == 0.0
        assert [bool(np.signbit(a[J0])) for a in log] == [True, True, False, False], runner


def test_kat_signed_zero_central(oracle):
    # per colour the plus point x1 and then the caller's x (the minus point).  Plus, colour 1: -0.0 + (+0.0) = +0.0.
    # Minus, colour 1: -0.0 - (+0.0) = -0.0 + -0.0 = -0.0 (the caller's zero survives); its restore -0.0 + (+0.0) = +0.0.
    # Colour 2 sees +0.0 in both points; colour 3 perturbs the component: +0.0 + eps3 > 0 and +0.0 - eps3 < 0.
    for r in _tridiag_runs(oracle, "central"):
        assert [bool(np.signbit(a[J0])) for a in r["args"]] == [False, True, False, False, False, True]


def test_kat_signed_zero_complex(oracle):
    # x1 .+ im*eps .* (colour .== k) adds (+0.0, eps) or (+0.0, +0.0) to every component: the real part of a -0.0 is
    # +0.0 in every call, the colour-3 call included (its imaginary part is eps there, +0.0 otherwise).
    colptr, rowval = tridiag_csc(N40)
    cv = cyc_colors(N40, 3)

    def f(fx, x):
        fx[:] = x
    logs = []
    log = []
    oracle.jacobian_complex(oracle.Problem.csc_same(N40, N40, colptr, rowval), np.zeros(len(rowval)), _recording(f, log),
                            _tridiag_x(), colorvec=cv)
    logs.append(log)
    log = []
    J = lit.CSC(N40, N40, colptr, rowval)
    lit.finite_difference_jacobian_complex(J, _recording(f, log), _tridiag_x(),
                                           dict(x1=np.zeros(N40, np.complex128), fx=np.zeros(N40, np.complex128)),
                                           colorvec=cv, sparsity=J)
    logs.append(log)
    eps = np.finfo(np.float64).eps
    for log in logs:
        assert [bool(np.signbit(a[J0].real)) for a in log] == [False, False, False]
        assert [a[J0].imag for a in log] == [0.0, 0.0, eps]


def test_kat_nan_component_gives_nan_step_of_its_colour_only(oracle):
    # norm of colour 2 is NaN, and Julia's max(NaN, absstep) is NaN: eps = [finite, NaN, finite].  Colour 2's J entries
    # are NaN; colours 1 and 3 see x1 + copysign(0, eps) = x1 in the NaN component, so their steps and values do not
    # change from the same x with that component set to anything finite.
    colptr, rowval = tridiag_csc(N40)
    cv = cyc_colors(N40, 3)
    x = np.random.default_rng(5).uniform(-2, 2, N40)
    x[1] = np.nan                                      # colour 2
    for fdtype in ("forward", "central"):
        J = lit.CSC(N40, N40, colptr, rowval)
        cache = dict(x1=np.zeros(N40), x2=np.zeros(N40), fx=np.zeros(N40), fx1=np.zeros(N40))
        rl = lit.finite_difference_jacobian(J, f_tridiag, x.copy(), cache, None, fdtype=fdtype, colorvec=cv, sparsity=J)
        ro = oracle.jacobian(oracle.Problem.csc_same(N40, N40, colptr, rowval), np.zeros(len(rowval)), f_tridiag, x.copy(),
                             fdtype=FD[fdtype], colorvec=cv)
        x_ok = x.copy()
        x_ok[1] = 1.0
        ro_ok = oracle.jacobian(oracle.Problem.csc_same(N40, N40, colptr, rowval), np.zeros(len(rowval)), f_tridiag, x_ok,
                                fdtype=FD[fdtype], colorvec=cv)
        for e in (ro["eps"], rl["eps"]):
            assert np.isfinite(e[0]) and np.isnan(e[1]) and np.isfinite(e[2]), (fdtype, e)
            assert e[0] == ro_ok["eps"][0] and e[2] == ro_ok["eps"][2]
        assert_same_bits(ro["eps"], rl["eps"], fdtype)
        assert np.isnan(J.nzval[colptr[1] - 1:colptr[2] - 1]).all()


def test_kat_inf_component_nan_count_per_call(oracle):
    # +Inf in component 1 (colour 2), forward.  f(x) and colour 1 see no NaN (x1 + Inf*false = x1 + 0.0).  Colour 2 adds
    # eps2 = Inf to its 13 components; the restore (x + Inf) - Inf makes all 13 NaN, so colour 3's call sees 13 NaNs.
    colptr, rowval = tridiag_csc(N40)
    cv = cyc_colors(N40, 3)
    x = np.random.default_rng(6).uniform(-2, 2, N40)
    x[1] = np.inf
    assert (cv == 2).sum() == 13
    logs = []
    log = []
    r = oracle.jacobian(oracle.Problem.csc_same(N40, N40, colptr, rowval), np.zeros(len(rowval)), _recording(f_tridiag, log),
                        x.copy(), colorvec=cv)
    assert r["eps"][1] == np.inf
    logs.append(log)
    log = []
    J = lit.CSC(N40, N40, colptr, rowval)
    cache = dict(x1=np.zeros(N40), x2=np.zeros(N40), fx=np.zeros(N40), fx1=np.zeros(N40))
    lit.finite_difference_jacobian(J, _recording(f_tridiag, log), x.copy(), cache, None, colorvec=cv, sparsity=J)
    logs.append(log)
    for log in logs:
        assert [int(np.isnan(a).sum()) for a in log] == [0, 0, 0, 13]


def test_kat_jvp_nan_step(oracle):
    # jvp.jl:252-253: sqrt(abs(dot(x, v))) is NaN when x holds a NaN, and max(NaN, absstep) keeps it
    x = np.array([1.0, np.nan, 2.0])
    v = np.array([0.5, 0.25, -1.0])
    for fdtype in (0, 1):
        r = oracle.jvp(lambda fx, xx: fx.__setitem__(slice(None), xx), x, v, 3, fdtype=fdtype)
        assert np.isnan(r["eps"])
