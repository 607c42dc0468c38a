"""Pins the CPU oracle against the known-answer fixtures of the reference's own tests
(tests/golden/kat_reference_tests.json, transcribed with file:line by tests/golden/make_golden.py).
CPU only. These read like test/coloring_tests.jl, test/cache_reuse_tests.jl and the Jacobian
block of test/finitedifftests.jl."""
import numpy as np
import pytest

from _util import (band_to_dense, csc_from_dense_pattern, csc_to_dense, f_tridiag, tridiag_csc,
                   tridiagonal_coo, tridiagonal_to_dense)

FDT = {"forward": 0, "central": 1}


class Counter:
    def __init__(self, f):
        self.f, self.calls, self.log = f, 0, []

    def __call__(self, fx, x):
        self.calls += 1
        self.log.append(x.copy())
        self.f(fx, x)


def test_default_relstep_and_epsilon(oracle, golden):
    g = golden["default_relstep"]
    assert oracle.default_relstep(0) == g["forward"]  # sqrt(eps)  epsilons.jl:137
    assert oracle.default_relstep(1) == g["central"]  # cbrt(eps)  epsilons.jl:139
    # epsilons.jl:26-29 / :50-53
    assert oracle.compute_epsilon(0, -4.0, 1e-3, 1e-8, 1.0) == 4e-3
    assert oracle.compute_epsilon(0, -4.0, 1e-3, 1e-8, -1.0) == -4e-3
    assert oracle.compute_epsilon(0, 0.0, 1e-3, 1e-8, 1.0) == 1e-8
    assert oracle.compute_epsilon(1, -4.0, 1e-3, 1e-8, -1.0) == 4e-3  # dir ignored for central


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_tridiag30_csc_same_pattern(oracle, golden, fdtype):
    # coloring_tests.jl:33-43 — CSC J, colorvec=repeat(1:3,10), cache-less entry, fcalls 4 / 6
    g = golden["tridiag30"]
    N = g["N"]
    colptr, rowval = tridiag_csc(N)
    P = oracle.Problem.csc_same(N, N, colptr, rowval)
    nz = np.full(len(rowval), np.nan)
    f = Counter(f_tridiag)
    x = np.array(g["x"])
    x0 = x.copy()
    r = oracle.jacobian(P, nz, f, x, fdtype=FDT[fdtype], colorvec=g["colorvec"], cacheless=True)
    assert r["fcalls"] == f.calls == g["fcalls"][fdtype]
    J = csc_to_dense(N, N, colptr, rowval, nz)
    np.testing.assert_allclose(J, np.array(g["J_expected"]), rtol=g["rtol"], atol=1e-7)
    np.testing.assert_allclose(x, x0, rtol=0, atol=1e-15)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_tridiag30_dense_J_csc_sparsity(oracle, golden, fdtype):
    # coloring_tests.jl:51-64 — dense J, sparsity=CSC
    g = golden["tridiag30"]
    N = g["N"]
    colptr, rowval = tridiag_csc(N)
    P = oracle.Problem.csc_to_dense(N, N, colptr, rowval)
    J = np.full(N * N, np.nan)
    f = Counter(f_tridiag)
    r = oracle.jacobian(P, J, f, np.array(g["x"]), fdtype=FDT[fdtype], colorvec=g["colorvec"], cacheless=True)
    assert r["fcalls"] == g["fcalls"][fdtype]
    np.testing.assert_allclose(J.reshape(N, N, order="F"), np.array(g["J_expected"]), rtol=g["rtol"], atol=1e-7)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_tridiag30_tridiagonal_coo(oracle, golden, fdtype):
    # coloring_tests.jl:72-82,94-96 — J::Tridiagonal goes through the generic COO hook
    g = golden["tridiag30"]
    N = g["N"]
    rows, cols, slots = tridiagonal_coo(N)
    P = oracle.Problem.coo_to_slots(N, N, rows, cols, slots, 3 * N - 2)
    buf = np.full(3 * N - 2, np.nan)
    r = oracle.jacobian(P, buf, Counter(f_tridiag), np.array(g["x"]), fdtype=FDT[fdtype],
                        colorvec=g["colorvec"], cacheless=True)
    assert r["fcalls"] == g["fcalls"][fdtype]
    np.testing.assert_allclose(tridiagonal_to_dense(N, buf), np.array(g["J_expected"]), rtol=g["rtol"], atol=1e-7)


def test_tridiag30_banded(oracle, golden):
    # coloring_tests.jl:90-92 — BandedMatrix(similar(J),(1,1))
    g = golden["tridiag30"]
    N = g["N"]
    P = oracle.Problem.banded(N, N, 1, 1)
    data = np.full(3 * N, np.nan)
    oracle.jacobian(P, data, f_tridiag, np.array(g["x"]), colorvec=g["colorvec"], cacheless=True)
    np.testing.assert_allclose(band_to_dense(N, N, 1, 1, data), np.array(g["J_expected"]), rtol=g["rtol"], atol=1e-7)


def f_lap5(g):
    def f(out, x):
        X = x.reshape(g, g, order="F")
        O = out.reshape(g, g, order="F")
        im = np.maximum(np.arange(g) - 1, 0)
        ip = np.minimum(np.arange(g) + 1, g - 1)
        O[:, :] = X + X[im, :] + X[ip, :] + X[:, im] + X[:, ip]
    return f


def lap5_pattern(g):
    """Structural pattern of the clamped 5-point stencil (coloring_tests.jl:99-108), as dense bool."""
    n = g * g
    A = np.zeros((n, n), bool)
    for j in range(g):
        for i in range(g):
            r = i + j * g
            for (a, b) in ((i, j), (max(i - 1, 0), j), (min(i + 1, g - 1), j), (i, max(j - 1, 0)), (i, min(j + 1, g - 1))):
                A[r, a + b * g] = True
    return A


def test_lap5_csc_vs_dense_columns(oracle):
    # coloring_tests.jl:99-119 shape (smaller grid): coloured CSC result == uncoloured dense result
    g = 12
    n = g * g
    A = lap5_pattern(g)
    colptr, rowval = csc_from_dense_pattern(A)
    colors = np.array([((i) + 2 * (j)) % 5 + 1 for j in range(g) for i in range(g)], dtype=np.int64)
    # distance-2 validity of the colouring: no row has two columns of one colour
    for r in range(n):
        cs = colors[np.nonzero(A[r])[0]]
        assert len(set(cs)) == len(cs)
    x = np.random.default_rng(3).random(n)
    nz = np.full(len(rowval), np.nan)
    r1 = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), nz, f_lap5(g), x.copy(), colorvec=colors,
                         cacheless=True)
    assert r1["fcalls"] == 6
    Jd = np.zeros(n * n)
    r2 = oracle.jacobian(oracle.Problem.dense(n, n), Jd, f_lap5(g), x.copy(), cacheless=True)
    assert r2["fcalls"] == n + 1
    np.testing.assert_allclose(csc_to_dense(n, n, colptr, rowval, nz), Jd.reshape(n, n, order="F"), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_nonsquare_4x8(oracle, golden, fdtype):
    # coloring_tests.jl:122-159 — 3-array cache ctor, fcalls = maxcolor+1 / 2*maxcolor, rtol 1e-6
    g = golden["nonsquare4x8"]
    n = g["n"]

    def f_nonsquare(y, x):
        x1, x2 = x[:n], x[n:]
        y[:] = (x1 - 3) ** 2 + x1 * x2 + (x2 + 4) ** 2 - 3

    import scipy.sparse as sp
    S = sp.csc_matrix((np.ones(2 * n), (np.array(g["rows"]) - 1, np.array(g["cols"]) - 1)), shape=(n, 2 * n))
    S.sort_indices()
    colptr, rowval = S.indptr.astype(np.int64) + 1, S.indices.astype(np.int64) + 1
    P = oracle.Problem.csc_same(n, 2 * n, colptr, rowval)
    nz = np.full(2 * n, np.nan)
    x0 = np.array(g["x0"])
    cache = dict(x1=x0.copy(), x2=np.zeros(2 * n), fx=np.zeros(n), fx1=np.zeros(n))
    f = Counter(f_nonsquare)
    r = oracle.jacobian(P, nz, f, x0.copy(), fdtype=FDT[fdtype], colorvec=g["colorvec"], cache=cache)
    assert r["fcalls"] == f.calls == g["fcalls"][fdtype]
    np.testing.assert_allclose(csc_to_dense(n, 2 * n, colptr, rowval, nz), np.array(g["J_analytic"]), rtol=g["rtol"])


def test_findstructralnz_order(oracle, golden):
    # coloring_tests.jl:163-168
    for case in golden["findstructralnz"]["cases"]:
        rows, cols = oracle.findstructralnz_dense(np.array(case["A"], dtype=float))
        assert rows.tolist() == case["rows"] and cols.tolist() == case["cols"]


_DENSE_FUNCS = {
    "_f": lambda dx, x: dx.__setitem__(slice(None), [x[0] ** 2 + x[1] ** 2, x[0] + x[1]]),
    "_f2": lambda dx, x: dx.__setitem__(slice(None), [x[0] ** 2 + x[1] ** 2, x[0]]),
    "_f3": lambda dx, x: dx.__setitem__(slice(None), [x[0] ** 2 + x[1] ** 2 - x[0]]),
    "_f4": lambda dx, x: dx.__setitem__(slice(None), [x[0] ** 2 + x[1] ** 2 - x[0], x[0] * x[1], x[0] * x[2], x[0]]),
    "_f5": lambda dx, x: dx.__setitem__(slice(None), [x[0] ** 2 + x[1] ** 2]),
}


def test_dense_prototype_sparsity(oracle, golden):
    # coloring_tests.jl:171-220 — sparsity is a dense 0/1 matrix; colorvec default 1:n; COO hook into dense J
    for case in golden["dense_prototypes"]["cases"]:
        S = np.array(case["sparsity"], dtype=float)
        m, n = S.shape
        rows, cols = oracle.findstructralnz_dense(S)
        P = oracle.Problem.coo_to_dense(m, n, rows, cols)
        J = np.zeros(m * n)
        theta = np.array(case["theta"])
        oracle.jacobian(P, J, _DENSE_FUNCS[case["name"]], theta.copy())
        np.testing.assert_allclose(J.reshape(m, n, order="F"), np.array(case["J"], dtype=float),
                                   rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_cache_reuse_poisoned(oracle, golden, fdtype):
    # cache_reuse_tests.jl:66-71 — poisoned x1/fx/fx1 must not leak into J (dense-column branch)
    g = golden["cache_reuse"]

    def foo(y, x):
        y[0], y[1], y[2] = 2 * x[0], 3 * x[1], 4 * x[0]

    P = oracle.Problem.dense(3, 2)
    cache = dict(x1=np.full(2, g["poison"]), x2=np.zeros(2), fx=np.full(3, g["poison"]), fx1=np.full(3, g["poison"]))
    J = np.zeros(6)
    oracle.jacobian(P, J, foo, np.array(g["X_TEST"]), fdtype=FDT[fdtype], cache=cache)
    np.testing.assert_allclose(J.reshape(3, 2, order="F"), np.array(g["J_REF"]), atol=g["atol"])


def test_central_sparse_leaves_x_unmutated(oracle, golden):
    # cache_reuse_tests.jl:73-83 — dense J + CSC sparsity, colorvec=1:2, central: x == x_orig afterwards
    g = golden["cache_reuse"]

    def foo(y, x):
        y[0], y[1], y[2] = 2 * x[0], 3 * x[1], 4 * x[0]

    colptr, rowval = csc_from_dense_pattern(np.array(g["J_REF"]))
    P = oracle.Problem.csc_to_dense(3, 2, colptr, rowval)
    cache = dict(x1=np.full(2, g["poison"]), x2=np.zeros(2), fx=np.full(3, g["poison"]), fx1=np.full(3, g["poison"]))
    J = np.zeros(6)
    x = np.array(g["X_TEST"])
    oracle.jacobian(P, J, foo, x, fdtype=1, cache=cache, colorvec=[1, 2])
    np.testing.assert_allclose(J.reshape(3, 2, order="F"), np.array(g["J_REF"]), atol=g["atol"])
    assert (x == np.array(g["X_TEST"])).all()


def _iipf(fvec, x):
    # finitedifftests.jl:399-402
    fvec[0] = (x[0] + 3) * (x[1] ** 3 - 7) + 18
    fvec[1] = np.sin(x[1] * np.exp(x[0]) - 1)


def _J_ref(x):
    # finitedifftests.jl:413
    return np.array([[-7 + x[1] ** 3, 3 * (3 + x[0]) * x[1] ** 2],
                     [np.exp(x[0]) * x[1] * np.cos(1 - np.exp(x[0]) * x[1]), np.exp(x[0]) * np.cos(1 - np.exp(x[0]) * x[1])]])


def test_analytic_2x2_bounds_dir_relstep_fin(oracle, golden):
    # finitedifftests.jl:447-463 (in-place block): forward<1e-6, central<1e-8, dir=-1, relstep kw, f_in
    g = golden["analytic2x2"]
    x = np.array(g["x"])
    Jref = _J_ref(x)
    P = oracle.Problem.dense(2, 2)

    def run(**kw):
        J = np.zeros(4)
        r = oracle.jacobian(P, J, kw.pop("f", _iipf), x.copy(), **kw)
        return J.reshape(2, 2, order="F"), r

    err = lambda a: np.max(np.abs(a - Jref))
    J, r = run()
    assert err(J) < g["bounds"]["forward"] and r["fcalls"] == 3
    J, _ = run(fdtype=1)
    assert err(J) < g["bounds"]["central"]
    J, _ = run(relstep=float(np.sqrt(np.finfo(float).eps)))
    assert err(J) < g["bounds"]["forward"]
    # f_in: no f(fx,x) call
    y = np.zeros(2)
    _iipf(y, x)
    J, r = run(f_in=y)
    assert err(J) < g["bounds"]["forward"] and r["fcalls"] == 2

    # dir=-1: the wrapped function errors if any component is perturbed upwards (finitedifftests.jl:409,456-457)
    def iipff(df, xx):
        if not np.all(xx <= x):
            raise AssertionError("perturbed upward")
        _iipf(df, xx)

    J, _ = run(f=iipff, dir=-1.0)
    assert err(J) < g["bounds"]["forward"]


def test_fcall_order_and_perturbation_central(oracle):
    # jacobians.jl:603-606 — central: f(fx1, x+eps) is called BEFORE f(fx, x-eps), colours ascending
    N = 9
    colptr, rowval = tridiag_csc(N)
    P = oracle.Problem.csc_same(N, N, colptr, rowval)
    x = np.linspace(1.0, 2.0, N)
    f = Counter(f_tridiag)
    r = oracle.jacobian(P, np.zeros(len(rowval)), f, x.copy(), fdtype=1, colorvec=np.tile([1, 2, 3], 3))
    assert f.calls == 6
    for k in range(3):
        up, dn = f.log[2 * k], f.log[2 * k + 1]
        mask = (np.arange(N) % 3) == k
        assert np.all(up[mask] > x[mask]) and np.all(dn[mask] < x[mask])
        np.testing.assert_allclose(up[~mask], x[~mask], rtol=0, atol=1e-15)
        np.testing.assert_allclose(up[mask] - x[mask], r["eps"][k], rtol=1e-7)


def test_empty_colour_still_calls_f(oracle):
    # jacobians.jl:547 — loop runs 1:maximum(colorvec); a colour with no columns still costs an f! call
    N = 6
    colptr, rowval = tridiag_csc(N)
    P = oracle.Problem.csc_same(N, N, colptr, rowval)
    colors = np.array([1, 2, 4, 1, 2, 4])  # colour 3 unused
    f = Counter(f_tridiag)
    nz = np.full(len(rowval), np.nan)
    r = oracle.jacobian(P, nz, f, np.linspace(1, 2, N), colorvec=colors)
    assert f.calls == 5
    assert np.isfinite(nz).all()
    # eps of the empty colour: norm(zeros)=0 -> eps = absstep = relstep
    assert r["eps"][2] == oracle.default_relstep(0)


def test_banded_whole_band_semantics(oracle):
    # ext/FiniteDiffBandedMatricesExt.jl:13-27 writes ALL in-band rows of a column: with fewer than l+u+1
    # colours the structurally-zero in-band slots receive values from same-coloured columns (SURVEY.md §3.3).
    g = 4
    n = g * g
    colors = np.array([((i) + 2 * (j)) % 5 + 1 for j in range(g) for i in range(g)], dtype=np.int64)
    x = np.random.default_rng(5).random(n)
    data = np.full((2 * g + 1) * n, np.nan)
    oracle.jacobian(oracle.Problem.banded(n, n, g, g), data, f_lap5(g), x.copy(), colorvec=colors)
    Jb = band_to_dense(n, n, g, g, data)
    A = lap5_pattern(g)
    # true nonzeros are right (compare with the uncoloured dense-column Jacobian)
    Jd = np.zeros(n * n)
    oracle.jacobian(oracle.Problem.dense(n, n), Jd, f_lap5(g), x.copy())
    np.testing.assert_allclose(Jb[A], Jd.reshape(n, n, order="F")[A], rtol=1e-6)
    # and at least one in-band structural zero received a spurious nonzero (documented trap)
    inband = np.abs(np.subtract.outer(np.arange(n), np.arange(n))) <= g
    assert np.any(np.abs(Jb[inband & ~A]) > 0.5)


def test_threads_match_single_thread(oracle):
    # OpenMP passes (used for the all-cores CPU baseline) give the same J when eps is pinned
    N = 3000
    colptr, rowval = tridiag_csc(N)
    P = oracle.Problem.csc_same(N, N, colptr, rowval)
    x = oracle.fill_x(N, 0x5EED + 2)
    cv = (np.arange(N) % 3) + 1
    a = np.zeros(len(rowval))
    r = oracle.jacobian(P, a, f_tridiag, x.copy(), colorvec=cv)
    b = np.zeros(len(rowval))
    oracle.jacobian(P, b, f_tridiag, x.copy(), colorvec=cv, nthreads=4, eps_override=r["eps"])
    assert (a == b).all()


def test_identity_map_all_fdtypes(oracle, golden):
    # finitedifftests.jl:600-605: J of (out, in) -> out .= in at ones(2), cache-less in-place call, every fdtype: J ≈ I
    g = golden["identity2"]
    x = np.array(g["x"])
    Jexp = np.array(g["J_expected"])

    def ident(out, xx):
        out[:] = xx

    for fd in g["fdtypes"]:
        J = np.full(4, np.nan)
        if fd == "complex":
            r = oracle.jacobian_complex(oracle.Problem.dense(2, 2), J, ident, x.copy())
            assert r["fcalls"] == 2
        else:
            r = oracle.jacobian(oracle.Problem.dense(2, 2), J, ident, x.copy(), fdtype=0 if fd == "forward" else 1)
            assert r["fcalls"] == (3 if fd == "forward" else 4)
        np.testing.assert_allclose(J.reshape(2, 2, order="F"), Jexp, rtol=g["rtol"], atol=g["rtol"])


def test_nonvector_input_identity(oracle, golden):
    # finitedifftests.jl:524-536: x = rand(2,2) (used as vec(x)), iipf(fx, x) = (fx .= x), J_ref = I(4); the in-place
    # cache-less call gets f_in = iipf(similar(x), x); max abs error < 1e-8 for every fdtype
    g = golden["nonvector_identity"]
    x = np.array(g["x"]).reshape(-1, order="F")          # Julia's vec(): column-major

    def ident(out, xx):
        out[:] = xx

    for fd in g["fdtypes"]:
        J = np.full(16, np.nan)
        if fd == "complex":
            r = oracle.jacobian_complex(oracle.Problem.dense(4, 4), J, ident, x.copy())
            assert r["fcalls"] == 4
        elif fd == "forward":
            r = oracle.jacobian(oracle.Problem.dense(4, 4), J, ident, x.copy(), fdtype=0, f_in=x.copy())
            assert r["fcalls"] == 4                       # f_in given: no f(x) evaluation (jacobians.jl:540-545)
        else:
            r = oracle.jacobian(oracle.Problem.dense(4, 4), J, ident, x.copy(), fdtype=1)
            assert r["fcalls"] == 8
        assert np.max(np.abs(J.reshape(4, 4, order="F") - np.eye(4))) < g["bound"]


@pytest.mark.parametrize("fdtype", [0, 1])
def test_no_drift_restores_exactly(oracle, fdtype):
    # no_drift (a test option, not the reference): every perturbed component is restored to its exact value, so each
    # colour's f! sees the pristine x outside its own colour.  The faithful run keeps the reference's (x1 + eps) - eps
    # drift, which with |x| up to 2 and a central step of about 1e-4 changes some components (the test has teeth).
    n = 200_000
    colptr, rowval = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    x0 = np.random.default_rng(3).uniform(-2, 2, n)
    P = oracle.Problem.csc_same(n, n, colptr, rowval)
    for no_drift in (True, False):
        x = x0.copy()
        r = oracle.jacobian(P, np.zeros(len(rowval)), f_tridiag, x, fdtype=fdtype, colorvec=cv, no_drift=no_drift)
        x1 = r["cache"]["x1"]
        if no_drift:
            assert np.array_equal(x1, x0) and np.array_equal(x, x0)
        elif fdtype == 1:
            assert not np.array_equal(x1, x0)
