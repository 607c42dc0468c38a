"""Complex-step colour loop (SURVEY.md §8f rank 1; src/jacobians.jl:623-648): oracle pinned on the reference tests'
complex-step fixtures (CPU), and the CUDA path bit-compared with the oracle (GPU)."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, band_to_dense, csc_from_dense_pattern, csc_to_dense, cyc_colors, tridiag_csc, tridiagonal_coo, tridiagonal_to_dense

EPS = np.finfo(float).eps


def f_tridiag_c(dx, x):
    n = len(x)
    dx[1:n - 1] = (x[0:n - 2] - 2 * x[1:n - 1]) + x[2:n]
    dx[0] = -2 * x[0] + x[1]
    dx[n - 1] = x[n - 2] - 2 * x[n - 1]


class Counter:
    def __init__(self, f):
        self.f, self.calls = f, 0

    def __call__(self, fx, x):
        self.calls += 1
        self.f(fx, x)


# ------------------------------------------------------------------------------------------------ oracle KATs (CPU)
def test_oracle_complex_tridiag30_all_J_kinds(oracle, golden):
    # coloring_tests.jl:45-49 (CSC, fcalls == 3), :66-70 (dense J + CSC sparsity), :84-88 (Tridiagonal)
    g = golden["tridiag30"]
    N = g["N"]
    Jexp = np.array(g["J_expected"])
    cv = g["colorvec"]
    x = np.array(g["x"])
    colptr, rowval = tridiag_csc(N)
    f = Counter(f_tridiag_c)
    nz = np.full(len(rowval), np.nan)
    r = oracle.jacobian_complex(oracle.Problem.csc_same(N, N, colptr, rowval), nz, f, x, colorvec=cv)
    assert r["fcalls"] == f.calls == 3
    np.testing.assert_allclose(csc_to_dense(N, N, colptr, rowval, nz), Jexp, rtol=1e-14, atol=1e-14)
    Jd = np.full(N * N, np.nan)
    r = oracle.jacobian_complex(oracle.Problem.csc_to_dense(N, N, colptr, rowval), Jd, f_tridiag_c, x, colorvec=cv)
    assert r["fcalls"] == 3
    np.testing.assert_allclose(Jd.reshape(N, N, order="F"), Jexp, rtol=1e-14, atol=1e-14)
    rows, cols, slots = tridiagonal_coo(N)
    buf = np.full(3 * N - 2, np.nan)
    oracle.jacobian_complex(oracle.Problem.coo_to_slots(N, N, rows, cols, slots, 3 * N - 2), buf, f_tridiag_c, x, colorvec=cv)
    np.testing.assert_allclose(tridiagonal_to_dense(N, buf), Jexp, rtol=1e-14, atol=1e-14)


def test_oracle_complex_analytic_2x2_and_nonsquare(oracle, golden):
    # finitedifftests.jl:462: err < 1e-14 with the complex cache (dense column branch, jacobians.jl:626-631)
    x = np.array(golden["analytic2x2"]["x"])

    def iipf(fvec, xx):
        fvec[0] = (xx[0] + 3) * (xx[1] ** 3 - 7) + 18
        fvec[1] = np.sin(xx[1] * np.exp(xx[0]) - 1)

    Jref = np.array([[-7 + x[1] ** 3, 3 * (3 + x[0]) * x[1] ** 2],
                     [np.exp(x[0]) * x[1] * np.cos(1 - np.exp(x[0]) * x[1]), np.exp(x[0]) * np.cos(1 - np.exp(x[0]) * x[1])]])
    J = np.zeros(4)
    r = oracle.jacobian_complex(oracle.Problem.dense(2, 2), J, iipf, x)
    assert r["fcalls"] == 2
    assert np.max(np.abs(J.reshape(2, 2, order="F") - Jref)) < 1e-14
    # coloring_tests.jl:122-159 non-square 4x8, two colours: fcalls == maximum(colorvec), rtol 1e-6
    g = golden["nonsquare4x8"]
    n = g["n"]

    def f_ns(y, xx):
        x1, x2 = xx[:n], xx[n:]
        y[:] = (x1 - 3) ** 2 + x1 * x2 + (x2 + 4) ** 2 - 3

    import scipy.sparse as sp
    S = sp.csc_matrix((np.ones(2 * n), (np.array(g["rows"]) - 1, np.array(g["cols"]) - 1)), shape=(n, 2 * n))
    S.sort_indices()
    colptr, rowval = S.indptr.astype(np.int64) + 1, S.indices.astype(np.int64) + 1
    nz = np.zeros(2 * n)
    r = oracle.jacobian_complex(oracle.Problem.csc_same(n, 2 * n, colptr, rowval), nz, f_ns, np.array(g["x0"]),
                                colorvec=g["colorvec"])
    assert r["fcalls"] == 2
    np.testing.assert_allclose(csc_to_dense(n, 2 * n, colptr, rowval, nz), np.array(g["J_analytic"]), rtol=1e-12)


def test_oracle_complex_poisoned_cache_shape(oracle, golden):
    # cache_reuse_tests.jl:57-71 (complex leg): J_REF = [2 0; 0 3; 4 0] through the dense column branch
    g = golden["cache_reuse"]

    def foo(y, x):
        y[0], y[1], y[2] = 2 * x[0], 3 * x[1], 4 * x[0]

    J = np.zeros(6)
    oracle.jacobian_complex(oracle.Problem.dense(3, 2), J, foo, np.array(g["X_TEST"]))
    np.testing.assert_allclose(J.reshape(3, 2, order="F"), np.array(g["J_REF"]), atol=1e-14)


def test_oracle_native_complex_tridiag_matches_python(oracle):
    N = 257
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    x = oracle.fill_x(N, 3)
    a = np.zeros(len(rowval))
    b = np.zeros(len(rowval))
    oracle.jacobian_complex(oracle.Problem.csc_same(N, N, colptr, rowval), a, f_tridiag_c, x, colorvec=cv)
    oracle.jacobian_complex(oracle.Problem.csc_same(N, N, colptr, rowval), b, oracle.native_fn("synth_tridiag_c"), x,
                            colorvec=cv, ctx=oracle.SynthTridiagCtx(N, 1))
    assert_same_bits(a, b, allow_nan=False)
    col_of = np.repeat(np.arange(1, N + 1), np.diff(colptr))
    assert_same_bits(a, np.where(rowval == col_of, -2.0, 1.0), allow_nan=False)           # (eps*k)/eps is exact


# ------------------------------------------------------------------------------------------------ CUDA path (GPU)
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


def _t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("strategy", [1, 2])
def test_gpu_complex_csc_bitexact(pkg, oracle, strategy):
    dev = torch.device("cuda:0")
    L = pkg._lib
    for N, colors in ((1000, 3), (4099, 7), (5, 3)):
        colptr, rowval = tridiag_csc(N)
        cv = cyc_colors(N, colors)
        x = torch.empty(N, dtype=torch.float64, device=dev)
        L.synth().fdbs_fill_x(x.data_ptr(), N, 0x5EED + 9, None)
        J = pkg.SparseMatrixCSC(N, N, _t64(colptr), _t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
        ctx = L.TridiagCtx(N, 0)
        f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag_c, C.c_void_p).value, ctx)
        cache = pkg.JacobianCache(x, "complex", colorvec=cv, sparsity=J, strategy=strategy)
        assert cache.fx1 is None and cache.fx.dtype == torch.complex128            # jacobians.jl:20-32
        x_before = x.clone()
        pkg.finite_difference_jacobian_(J, f, x, cache)
        torch.cuda.synchronize()
        assert_same_bits(x, x_before, allow_nan=False)
        assert ctx.calls == colors                                                  # coloring_tests.jl:48: fcalls == 3
        np.testing.assert_array_equal(cache._last_plan.eps(), np.full(colors, EPS))
        ref = np.full(len(rowval), np.nan)
        r = oracle.jacobian_complex(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag_c"),
                                    oracle.fill_x(N, 0x5EED + 9), colorvec=cv, ctx=oracle.SynthTridiagCtx(N, 1))
        assert r["fcalls"] == colors
        assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)


@pytest.mark.gpu
def test_gpu_complex_kats_python_callbacks(pkg, golden):
    dev = torch.device("cuda:0")
    g = golden["tridiag30"]
    N = g["N"]
    Jexp = np.array(g["J_expected"])
    cv = np.array(g["colorvec"], dtype=np.int64)
    x = torch.tensor(g["x"], dtype=torch.float64, device=dev)
    colptr, rowval = tridiag_csc(N)
    sp = pkg.SparseMatrixCSC(N, N, _t64(colptr), _t64(rowval), torch.zeros(len(rowval), dtype=torch.float64, device=dev))

    def f_t(dx, xx):
        assert xx.dtype == torch.complex128
        n = xx.numel()
        dx[1:n - 1] = (xx[0:n - 2] - 2 * xx[1:n - 1]) + xx[2:n]
        dx[0] = -2 * xx[0] + xx[1]
        dx[n - 1] = xx[n - 2] - 2 * xx[n - 1]

    f = Counter(f_t)
    J = sp.similar()
    J.nzval.fill_(float("nan"))
    pkg.finite_difference_jacobian_(J, f, x, "complex", colorvec=cv)                 # cache-less, Val{:complex}
    assert f.calls == 3                                                               # coloring_tests.jl:45-49
    np.testing.assert_allclose(J.to_dense(), Jexp, rtol=1e-14, atol=1e-14)
    Jd = pkg.zeros_colmajor(N, N, dev)
    pkg.finite_difference_jacobian_(Jd, Counter(f_t), x, "complex", colorvec=cv, sparsity=sp)   # :66-70
    np.testing.assert_allclose(Jd.cpu().numpy(), Jexp, rtol=1e-14, atol=1e-14)
    Jt = pkg.Tridiagonal(N, device=dev)
    pkg.finite_difference_jacobian_(Jt, Counter(f_t), x, "complex", colorvec=cv)      # :84-88
    np.testing.assert_allclose(Jt.to_dense(), Jexp, rtol=1e-14, atol=1e-14)
    Jb = pkg.BandedMatrix(N, N, 1, 1, device=dev)
    pkg.finite_difference_jacobian_(Jb, Counter(f_t), x, "complex", colorvec=cv)
    np.testing.assert_allclose(Jb.to_dense(), Jexp, rtol=1e-14, atol=1e-14)
    # analytic 2x2, dense column branch, err < 1e-14 (finitedifftests.jl:462)
    xa = torch.tensor(golden["analytic2x2"]["x"], dtype=torch.float64, device=dev)
    xh = np.array(golden["analytic2x2"]["x"])

    def iipf(fvec, xx):
        fvec[0] = (xx[0] + 3) * (xx[1] ** 3 - 7) + 18
        fvec[1] = torch.sin(xx[1] * torch.exp(xx[0]) - 1)

    Jref = np.array([[-7 + xh[1] ** 3, 3 * (3 + xh[0]) * xh[1] ** 2],
                     [np.exp(xh[0]) * xh[1] * np.cos(1 - np.exp(xh[0]) * xh[1]), np.exp(xh[0]) * np.cos(1 - np.exp(xh[0]) * xh[1])]])
    J2 = pkg.zeros_colmajor(2, 2, dev)
    pkg.finite_difference_jacobian_(J2, iipf, xa, pkg.JacobianCache(xa, "complex"))
    assert np.max(np.abs(J2.cpu().numpy() - Jref)) < 1e-13
