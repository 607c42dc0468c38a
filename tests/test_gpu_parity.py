"""GPU parity tests (run with -m gpu on an H100).  Everything goes through the C ABI (libfdjac_b200.so) via the
host-side mirror; the CPU oracle is only the checker.

Bars: index / colour / f!-call parity exact; Jacobian values BIT-EXACT against the oracle when it is fed the
device-computed step sizes (same IEEE subtraction/division, bit-identical synthetic f!); device eps vs oracle eps
within 1e-14 relative (reduction order differs; Julia's own norm is OpenBLAS dnrm2 — bit-level eps is unpinned);
against closed-form answers the reference tests' own tolerances (1e-6 forward, 1e-8 central, rtol sqrt(eps))."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import (assert_same_bits, csc_from_dense_pattern, cyc_colors, fdb_env, tridiag_csc)  # noqa: E402

# FDB_SM_COUNT=k: grids sized as if the device had k SMs, so the tile loops take several steps per block at test sizes
SM_COUNTS = [None, 1, 3]

FD = {"forward": 0, "central": 1}


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def native(pkg, name, ctx, max_batch=1):
    return pkg.NativeFn(C.cast(getattr(pkg._lib.synth(), name), C.c_void_p).value, ctx, max_batch=max_batch)


def dev_x(pkg, dev, n, seed):
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, seed, None)
    torch.cuda.synchronize()
    return x


def t64(a, device=None):
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64))
    return t.to(device) if device is not None else t


def run_csc_tridiag(pkg, oracle, dev, N, fdtype, *, no_drift=False, max_batch=1, scratch_bytes=0, index_on_device=False,
                    colors=3, strategy=0):
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, colors)
    x = dev_x(pkg, dev, N, 0x5EED + 2)
    idev = dev if index_on_device else None
    J = pkg.SparseMatrixCSC(N, N, t64(colptr, idev), t64(rowval, idev),
                            torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
    ctx = pkg._lib.TridiagCtx(N, 0)
    f = native(pkg, "fdbs_tridiag", ctx, max_batch)
    cache = pkg.JacobianCache(x, fdtype, colorvec=t64(cv, idev) if index_on_device else cv, sparsity=J,
                              no_drift=no_drift, max_batch=max_batch, scratch_bytes=scratch_bytes, strategy=strategy)
    x_before = x.clone()
    pkg.finite_difference_jacobian_(J, f, x, cache)
    torch.cuda.synchronize()
    assert_same_bits(x, x_before, "caller's x must be untouched", allow_nan=False)
    plan = cache._last_plan
    eps = plan.eps()
    xh = oracle.fill_x(N, 0x5EED + 2)
    assert_same_bits(xh, x.cpu().numpy(), allow_nan=False)
    ref = np.full(len(rowval), np.nan)
    r = oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"), xh,
                        fdtype=FD[fdtype], colorvec=cv, eps_override=eps, no_drift=no_drift,
                        ctx=oracle.SynthTridiagCtx(N, 1))
    own = oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), np.zeros(len(rowval)),
                          oracle.native_fn("synth_tridiag"), xh.copy(), fdtype=FD[fdtype], colorvec=cv,
                          ctx=oracle.SynthTridiagCtx(N, 1))
    return J.nzval.cpu().numpy(), ref, eps, own["eps"], ctx.calls, r["fcalls"], plan


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("no_drift", [False, True])
def test_c1_tridiag_csc_bitexact(pkg, oracle, dev, fdtype, no_drift):
    """BASELINE config C1: N=1000 tridiagonal, colorvec=repeat(1:3), CSC J (coloring_tests.jl:33-43 shape)."""
    got, ref, eps, eps_o, calls, ocalls, plan = run_csc_tridiag(pkg, oracle, dev, 1000, fdtype, no_drift=no_drift)
    assert calls == ocalls == (4 if fdtype == "forward" else 6)
    np.testing.assert_allclose(eps, eps_o, rtol=1e-14, atol=0)
    assert_same_bits(got, ref, allow_nan=False)
    info = plan.info()
    assert info["n_groups"] == 1 and info["n_colors"] == 3 and info["n_entries"] == 2998
    assert info["alg_bytes_scatter"] == 32 * 2998 + 16 * 1000 + 8


@pytest.mark.parametrize("N", [1, 2, 3, 5, 31, 257, 4099])
def test_tridiag_ragged_sizes(pkg, oracle, dev, N):
    for fdtype in ("forward", "central"):
        got, ref, *_ = run_csc_tridiag(pkg, oracle, dev, N, fdtype)
        assert_same_bits(got, ref, allow_nan=False)


def test_tridiag_index_arrays_on_device(pkg, oracle, dev):
    got, ref, *_ = run_csc_tridiag(pkg, oracle, dev, 5000, "forward", index_on_device=True)
    assert_same_bits(got, ref, allow_nan=False)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_tridiag_multi_group_and_batch(pkg, oracle, dev, fdtype):
    # 7 colours, scratch budget for ~2 slabs -> several scatter launches; batched f! (3 points per callback)
    N = 20000
    small = 8 * (N + 2) * (4 if fdtype == "central" else 2) + 64
    a = run_csc_tridiag(pkg, oracle, dev, N, fdtype, colors=7, scratch_bytes=small, strategy=1)   # fused pass per group
    assert a[6].info()["n_groups"] > 1 and a[6].info()["strategy"] == 0
    assert_same_bits(a[0], a[1], allow_nan=False)
    a = run_csc_tridiag(pkg, oracle, dev, N, fdtype, colors=7, scratch_bytes=small)               # auto -> column lists
    assert a[6].info()["n_groups"] > 1 and a[6].info()["strategy"] == 1
    assert_same_bits(a[0], a[1], allow_nan=False)
    b = run_csc_tridiag(pkg, oracle, dev, N, fdtype, colors=7, max_batch=3)
    assert_same_bits(b[0], b[1], allow_nan=False)
    assert b[4] == b[5]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_per_colour_list_strategy_tridiag(pkg, oracle, dev, fdtype):
    # strategy 2: per-colour column lists (ext/FiniteDiffSparseArraysExt.jl:38-47 shape), several colours per launch,
    # more colours than kMaxSegs, odd sizes, batched f!
    for N, colors, mb in ((4099, 3, 1), (10000, 19, 1), (10000, 19, 4), (7, 3, 1)):
        got, ref, eps, eps_o, calls, ocalls, plan = run_csc_tridiag(pkg, oracle, dev, N, fdtype, colors=colors, strategy=2,
                                                                    max_batch=mb)
        assert plan.info()["strategy"] == 1 and calls == ocalls
        assert_same_bits(got, ref, allow_nan=False)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_unaligned_buffers_take_scalar_paths(pkg, oracle, dev, fdtype):
    # x and nzval only 8-byte aligned (views at an odd offset): the 16-byte vector paths must fall back, same bits
    _unaligned_case(pkg, oracle, dev, fdtype, 5003)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("N,sm_count", [(5003, 1), (5003, 3), (300_001, 1), (300_001, 3)])
def test_unaligned_buffers_multiwave(pkg, oracle, dev, fdtype, N, sm_count):
    # the same scalar paths with several tiles per block
    _unaligned_case(pkg, oracle, dev, fdtype, N, sm_count)


def _unaligned_case(pkg, oracle, dev, fdtype, N, sm_count=None):
    from _util import f_tridiag
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    xbuf = torch.zeros(N + 1, dtype=torch.float64, device=dev)
    x = xbuf[1:]
    x.copy_(dev_x(pkg, dev, N, 41))
    assert x.data_ptr() % 16 == 8
    nzbuf = torch.full((len(rowval) + 1,), float("nan"), dtype=torch.float64, device=dev)
    J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), nzbuf[1:])
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
    with fdb_env(SM_COUNT=sm_count):
        pkg.finite_difference_jacobian_(J, f_tridiag_t, x, cache)
    ref = np.full(len(rowval), np.nan)
    oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, f_tridiag, oracle.fill_x(N, 41), fdtype=FD[fdtype],
                    colorvec=cv, eps_override=cache._last_plan.eps())
    assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_cuda_graph_replay(pkg, oracle, dev, fdtype):
    # use_graph: the call is captured once and replayed; results stay bit-identical, counters advance per replay,
    # a change of buffers re-captures
    N = 50000
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
    ctx = pkg._lib.TridiagCtx(N, 0)
    f = native(pkg, "fdbs_tridiag", ctx)
    x = dev_x(pkg, dev, N, 31)
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J, use_graph=True)
    per_call = 4 if fdtype == "forward" else 6
    for it in range(3):
        J.nzval.fill_(float("nan"))
        pkg.finite_difference_jacobian_(J, f, x, cache)
        torch.cuda.synchronize()
        ref = np.full(len(rowval), np.nan)
        oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"),
                        oracle.fill_x(N, 31), fdtype=FD[fdtype], colorvec=cv, eps_override=cache._last_plan.eps(),
                        ctx=oracle.SynthTridiagCtx(N, 1))
        assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)
        c = cache._last_plan.counters()
        assert c["jacobians"] == it + 1 and c["f_points"] == per_call * (it + 1)
    assert ctx.calls == per_call            # the callback itself ran only during the capture
    # new x buffer with new values -> re-capture, correct result for the new point
    x2 = dev_x(pkg, dev, N, 32)
    pkg.finite_difference_jacobian_(J, f, x2, cache)
    torch.cuda.synchronize()
    ref = np.full(len(rowval), np.nan)
    oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"),
                    oracle.fill_x(N, 32), fdtype=FD[fdtype], colorvec=cv, eps_override=cache._last_plan.eps(),
                    ctx=oracle.SynthTridiagCtx(N, 1))
    assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)
    assert ctx.calls == 2 * per_call
    # in-place update of the SAME x buffer: the replay picks up the new values (eps is recomputed on the device)
    x2.copy_(x)
    pkg.finite_difference_jacobian_(J, f, x2, cache)
    torch.cuda.synchronize()
    oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"),
                    oracle.fill_x(N, 31), fdtype=FD[fdtype], colorvec=cv, eps_override=cache._last_plan.eps(),
                    ctx=oracle.SynthTridiagCtx(N, 1))
    assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)
    assert ctx.calls == 2 * per_call


def test_c2_full_size_bitexact(pkg, oracle, dev):
    """BASELINE config C2 at full size: N=10^7 tridiagonal, 3 colours, forward and central, CSC J — bit-compared
    with the CPU oracle, plus the size-independent property that the Jacobian of the linear stencil is the stencil."""
    N = 10_000_000
    for fdtype, tol in (("forward", 1e-6), ("central", 1e-8)):
        got, ref, eps, eps_o, calls, ocalls, plan = run_csc_tridiag(pkg, oracle, dev, N, fdtype)
        assert calls == ocalls
        np.testing.assert_allclose(eps, eps_o, rtol=1e-13)
        assert_same_bits(got, ref, allow_nan=False)
        colptr, rowval = tridiag_csc(N)
        col_of = np.repeat(np.arange(1, N + 1), np.diff(colptr))
        expected = np.where(rowval == col_of, -2.0, 1.0)
        assert np.max(np.abs(got - expected)) < tol
        del got, ref


# ---------------------------------------------------------------- reference KATs through the Python mirror (torch f!)
def f_tridiag_t(dx, x):
    n = x.numel()
    dx[1:n - 1] = (x[0:n - 2] - 2 * x[1:n - 1]) + x[2:n]
    dx[0] = -2 * x[0] + x[1]
    dx[n - 1] = x[n - 2] - 2 * x[n - 1]


class Counter:
    def __init__(self, f):
        self.f, self.calls, self.log = f, 0, []

    def __call__(self, fx, x):
        self.calls += 1
        self.log.append(x.clone())
        self.f(fx, x)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_kat_tridiag30_all_J_kinds(pkg, golden, dev, fdtype):
    # coloring_tests.jl:33-43 (CSC), :51-64 (dense J + CSC sparsity), :72-82 (Tridiagonal), :90-92 (Banded)
    g = golden["tridiag30"]
    N = g["N"]
    Jexp = np.array(g["J_expected"])
    cv = np.array(g["colorvec"], dtype=np.int64)
    x = torch.tensor(g["x"], dtype=torch.float64, device=dev)
    colptr, rowval = tridiag_csc(N)
    sp = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.zeros(len(rowval), dtype=torch.float64, device=dev))
    ncalls = g["fcalls"][fdtype]

    f = Counter(f_tridiag_t)
    J = sp.similar()
    J.nzval.fill_(float("nan"))
    pkg.finite_difference_jacobian_(J, f, x, fdtype, colorvec=cv)
    assert f.calls == ncalls
    np.testing.assert_allclose(J.to_dense(), Jexp, rtol=g["rtol"], atol=1e-7)

    f = Counter(f_tridiag_t)
    Jd = pkg.zeros_colmajor(N, N, dev)
    Jd.fill_(float("nan"))
    pkg.finite_difference_jacobian_(Jd, f, x, fdtype, colorvec=cv, sparsity=sp)
    assert f.calls == ncalls
    np.testing.assert_allclose(Jd.cpu().numpy(), Jexp, rtol=g["rtol"], atol=1e-7)

    f = Counter(f_tridiag_t)
    Jt = pkg.Tridiagonal(N, device=dev)
    Jt.buf.fill_(float("nan"))
    pkg.finite_difference_jacobian_(Jt, f, x, fdtype, colorvec=cv)
    assert f.calls == ncalls
    np.testing.assert_allclose(Jt.to_dense(), Jexp, rtol=g["rtol"], atol=1e-7)

    Jb = pkg.BandedMatrix(N, N, 1, 1, device=dev)
    Jb.data.fill_(float("nan"))
    pkg.finite_difference_jacobian_(Jb, Counter(f_tridiag_t), x, fdtype, colorvec=cv)
    np.testing.assert_allclose(Jb.to_dense(), Jexp, rtol=g["rtol"], atol=1e-7)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_kat_nonsquare_4x8(pkg, golden, dev, fdtype):
    # coloring_tests.jl:122-159
    g = golden["nonsquare4x8"]
    n = g["n"]

    def f_nonsquare(y, x):
        x1, x2 = x[:n], x[n:]
        y[:] = (x1 - 3) ** 2 + x1 * x2 + (x2 + 4) ** 2 - 3

    import scipy.sparse as sps
    S = sps.csc_matrix((np.ones(2 * n), (np.array(g["rows"]) - 1, np.array(g["cols"]) - 1)), shape=(n, 2 * n))
    sparsity = pkg.SparseMatrixCSC.from_scipy(S, dev)
    x0 = torch.tensor(g["x0"], dtype=torch.float64, device=dev)
    y0 = torch.zeros(n, dtype=torch.float64, device=dev)
    cache = pkg.JacobianCache(x0.clone(), y0.clone(), y0.clone(), fdtype, sparsity=sparsity,
                              colorvec=np.array(g["colorvec"], dtype=np.int64))
    f = Counter(f_nonsquare)
    J = sparsity.similar()
    pkg.finite_difference_jacobian_(J, f, x0, cache)
    assert f.calls == g["fcalls"][fdtype]
    np.testing.assert_allclose(J.to_dense(), np.array(g["J_analytic"]), rtol=g["rtol"])


def test_kat_dense_prototypes(pkg, golden, dev):
    # coloring_tests.jl:171-220
    funcs = {
        "_f": lambda dx, x: dx.copy_(torch.stack([x[0] ** 2 + x[1] ** 2, x[0] + x[1]])),
        "_f2": lambda dx, x: dx.copy_(torch.stack([x[0] ** 2 + x[1] ** 2, x[0]])),
        "_f3": lambda dx, x: dx.copy_(torch.stack([x[0] ** 2 + x[1] ** 2 - x[0]])),
        "_f4": lambda dx, x: dx.copy_(torch.stack([x[0] ** 2 + x[1] ** 2 - x[0], x[0] * x[1], x[0] * x[2], x[0]])),
        "_f5": lambda dx, x: dx.copy_(torch.stack([x[0] ** 2 + x[1] ** 2])),
    }
    for case in golden["dense_prototypes"]["cases"]:
        S = np.array(case["sparsity"])
        m, n = S.shape
        theta = torch.tensor(case["theta"], dtype=torch.float64, device=dev)
        y0 = torch.zeros(m, dtype=torch.float64, device=dev)
        J = pkg.zeros_colmajor(m, n, dev)
        cache = pkg.JacobianCache(theta.clone(), y0.clone(), y0.clone(), "forward", sparsity=S)
        pkg.finite_difference_jacobian_(J, funcs[case["name"]], theta, cache)
        np.testing.assert_allclose(J.cpu().numpy(), np.array(case["J"], dtype=float), rtol=1e-6, atol=1e-6)


def _foo(y, x):
    y[0], y[1], y[2] = 2 * x[0], 3 * x[1], 4 * x[0]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_kat_cache_reuse_poisoned(pkg, golden, dev, fdtype):
    # cache_reuse_tests.jl:57-71
    g = golden["cache_reuse"]
    X = torch.tensor(g["X_TEST"], dtype=torch.float64, device=dev)
    P = g["poison"]
    cache = pkg.JacobianCache(torch.full((2,), P, dtype=torch.float64, device=dev),
                              torch.full((3,), P, dtype=torch.float64, device=dev),
                              torch.full((3,), P, dtype=torch.float64, device=dev), fdtype)
    J = pkg.zeros_colmajor(3, 2, dev)
    pkg.finite_difference_jacobian_(J, _foo, X, cache)
    np.testing.assert_allclose(J.cpu().numpy(), np.array(g["J_REF"]), atol=g["atol"])
    # fresh cache reused at a new x (:57-64)
    cache = pkg.JacobianCache(torch.zeros(2, dtype=torch.float64, device=dev),
                              torch.zeros(3, dtype=torch.float64, device=dev), fdtype)
    pkg.finite_difference_jacobian_(J, _foo, torch.zeros(2, dtype=torch.float64, device=dev), cache)
    J.zero_()
    pkg.finite_difference_jacobian_(J, _foo, X, cache)
    np.testing.assert_allclose(J.cpu().numpy(), np.array(g["J_REF"]), atol=g["atol"])


def test_kat_central_sparse_leaves_x_unmutated(pkg, golden, dev):
    # cache_reuse_tests.jl:73-83
    g = golden["cache_reuse"]
    spJ = pkg.SparseMatrixCSC.from_scipy(np.array(g["J_REF"]) != 0, dev)
    P = g["poison"]
    cache = pkg.JacobianCache(torch.full((2,), P, dtype=torch.float64, device=dev),
                              torch.full((3,), P, dtype=torch.float64, device=dev),
                              torch.full((3,), P, dtype=torch.float64, device=dev), "central")
    J = pkg.zeros_colmajor(3, 2, dev)
    x = torch.tensor(g["X_TEST"], dtype=torch.float64, device=dev)
    x_orig = x.clone()
    pkg.finite_difference_jacobian_(J, _foo, x, cache, sparsity=spJ, colorvec=range(1, 3))
    np.testing.assert_allclose(J.cpu().numpy(), np.array(g["J_REF"]), atol=g["atol"])
    assert_same_bits(x, x_orig, allow_nan=False)


def test_kat_analytic_2x2(pkg, golden, dev):
    # finitedifftests.jl:398-463 (in-place block)
    g = golden["analytic2x2"]
    xh = np.array(g["x"])
    x = torch.tensor(xh, dtype=torch.float64, device=dev)

    def iipf(fvec, xx):
        fvec[0] = (xx[0] + 3) * (xx[1] ** 3 - 7) + 18
        fvec[1] = torch.sin(xx[1] * torch.exp(xx[0]) - 1)

    Jref = np.array([[-7 + xh[1] ** 3, 3 * (3 + xh[0]) * xh[1] ** 2],
                     [np.exp(xh[0]) * xh[1] * np.cos(1 - np.exp(xh[0]) * xh[1]), np.exp(xh[0]) * np.cos(1 - np.exp(xh[0]) * xh[1])]])
    err = lambda J: float(np.max(np.abs(J.cpu().numpy() - Jref)))
    fwd, cen = pkg.JacobianCache(x, "forward"), pkg.JacobianCache(x, "central")
    assert list(fwd.colorvec) == [1, 2]                    # finitedifftests.jl:420
    J = pkg.zeros_colmajor(2, 2, dev)
    pkg.finite_difference_jacobian_(J, iipf, x, fwd)
    assert err(J) < g["bounds"]["forward"]
    pkg.finite_difference_jacobian_(J, iipf, x, cen)
    assert err(J) < g["bounds"]["central"]
    pkg.finite_difference_jacobian_(J, iipf, x, "central")          # cache-less, Val{:central}
    assert err(J) < g["bounds"]["central"]
    pkg.finite_difference_jacobian_(J, iipf, x, fwd, relstep=float(np.sqrt(np.finfo(float).eps)))
    assert err(J) < g["bounds"]["forward"]
    y = torch.zeros(2, dtype=torch.float64, device=dev)
    iipf(y, x)
    f = Counter(iipf)
    pkg.finite_difference_jacobian_(J, f, x, fwd, y)
    assert err(J) < g["bounds"]["forward"] and f.calls == 2

    def iipff(df, xx):                                               # finitedifftests.jl:409
        if not bool(torch.all(xx <= x)):
            raise RuntimeError("perturbed upward")
        iipf(df, xx)

    pkg.finite_difference_jacobian_(J, iipff, x, fwd, dir=-1)
    assert err(J) < g["bounds"]["forward"]
    with pytest.raises(RuntimeError, match="perturbed upward"):      # @test_throws Any  :457
        pkg.finite_difference_jacobian_(J, iipff, x, fwd)


def test_matrix_shaped_x(pkg, dev):
    # finitedifftests.jl:516-528: x is a 2x2 matrix, f = identity -> J = I(4)
    x = torch.rand(2, 2, dtype=torch.float64, device=dev)
    J = pkg.zeros_colmajor(4, 4, dev)
    pkg.finite_difference_jacobian_(J, lambda fx, xx: fx.copy_(xx), x, "forward")
    assert np.max(np.abs(J.cpu().numpy() - np.eye(4))) < 1e-8
    pkg.finite_difference_jacobian_(J, lambda fx, xx: fx.copy_(xx), x, "central")
    assert np.max(np.abs(J.cpu().numpy() - np.eye(4))) < 1e-8


# ---------------------------------------------------------------- other structures, bit-exact vs the oracle
def lap5_colors(g):
    return np.array([((i) + 2 * (j)) % 5 + 1 for j in range(g) for i in range(g)], dtype=np.int64)


def lap5_csc(g):
    import scipy.sparse as sps
    n = g * g
    idx = np.arange(n)
    i, j = idx % g, idx // g
    cols = [idx, np.maximum(i - 1, 0) + j * g, np.minimum(i + 1, g - 1) + j * g, i + np.maximum(j - 1, 0) * g,
            i + np.minimum(j + 1, g - 1) * g]
    A = sps.csc_matrix((np.ones(5 * n), (np.tile(idx, 5), np.concatenate(cols))), shape=(n, n))
    A.sum_duplicates()
    A.sort_indices()
    return A


@pytest.mark.parametrize("g", [120, 121])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_lap5_csc_and_banded_bitexact(pkg, oracle, dev, fdtype, g):
    """2-D 5-point stencil (coloring_tests.jl:99-108 shape; BASELINE config C3 at reduced g): CSC path and the
    whole-band BandedMatrix path (ext/FiniteDiffBandedMatricesExt.jl:13-27, incl. its spurious in-band entries)."""
    # even and odd band half-widths (the flat-stream band kernel cuts the band storage into 16-byte aligned chunks)
    n = g * g
    A = lap5_csc(g)
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    cv = lap5_colors(g)
    x = dev_x(pkg, dev, n, 0x5EED + 3)
    xh = oracle.fill_x(n, 0x5EED + 3)
    # CSC
    J = pkg.SparseMatrixCSC(n, n, t64(colptr), t64(rowval), torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
    ctx = pkg._lib.Lap5Ctx(g, 0)
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_lap5", ctx), x, cache)
    eps = cache._last_plan.eps()
    ref = np.full(A.nnz, np.nan)
    r = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_lap5"), xh.copy(),
                        fdtype=FD[fdtype], colorvec=cv, eps_override=eps, ctx=oracle.SynthLap5Ctx(g, 1))
    assert ctx.calls == r["fcalls"]
    assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)
    # Banded l=u=g, 5 colours: whole-band fill
    Jb = pkg.BandedMatrix(n, n, g, g, device=dev)
    Jb.data.fill_(float("nan"))
    cache_b = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=Jb)
    pkg.finite_difference_jacobian_(Jb, native(pkg, "fdbs_lap5", pkg._lib.Lap5Ctx(g, 0)), x, cache_b)
    refb = np.full((2 * g + 1) * n, np.nan)
    oracle.jacobian(oracle.Problem.banded(n, n, g, g), refb, oracle.native_fn("synth_lap5"), xh.copy(),
                    fdtype=FD[fdtype], colorvec=cv, eps_override=cache_b._last_plan.eps(), ctx=oracle.SynthLap5Ctx(g, 1))
    assert_same_bits(Jb.data.cpu().numpy(), refb, allow_nan=False)
    # banded sparsity scattered into a dense J
    if g <= 120:
        Jd = pkg.zeros_colmajor(n, n, dev)
        cache_d = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=Jb)
        pkg.finite_difference_jacobian_(Jd, native(pkg, "fdbs_lap5", pkg._lib.Lap5Ctx(g, 0)), x, cache_d)
        refd = np.zeros(n * n)
        oracle.jacobian(oracle.Problem.banded_to_dense(n, n, g, g), refd, oracle.native_fn("synth_lap5"), xh.copy(),
                        fdtype=FD[fdtype], colorvec=cv, eps_override=cache_d._last_plan.eps(), ctx=oracle.SynthLap5Ctx(g, 1))
        assert_same_bits(Jd.cpu().numpy().reshape(-1, order="F"), refd, allow_nan=False)


NARROW_BANDS = [(30, 30, 1, 1), (50, 40, 3, 0), (40, 50, 0, 2), (17, 17, 16, 16), (300, 200, 70, 10), (200, 300, 5, 90),
                (130, 130, 129, 129)]


def test_narrow_band_and_rectangular_band(pkg, oracle, dev):
    # narrow-band tiling branch (w=3), non-square m != n, unequal l/u
    # (the last three take the warp-per-column wide-band kernel, l+u+1 >= 64)
    _narrow_bands(pkg, oracle, dev, NARROW_BANDS)


@pytest.mark.parametrize("sm_count", SM_COUNTS)
def test_narrow_band_multiwave(pkg, oracle, dev, sm_count):
    # the same shapes with several tiles per block, plus two long bands (w = 3, 5) that give every block of the tiled
    # kernel several tiles at sm_count = 1
    _narrow_bands(pkg, oracle, dev, NARROW_BANDS + [(60000, 70000, 1, 1), (50000, 40000, 3, 1)], sm_count)


def _narrow_bands(pkg, oracle, dev, shapes, sm_count=None):
    for (m, n, l, u) in shapes:
        cv = cyc_colors(n, l + u + 1)
        x = dev_x(pkg, dev, n, 77)
        xh = oracle.fill_x(n, 77)

        def f_t(fx, xx, m=m, n=n):
            k = min(m, n)
            fx.zero_()
            fx[:k] = xx[:k] * xx[:k]
            fx[1:k] += 0.5 * xx[: k - 1]

        def f_n(fx, xx, m=m, n=n):
            k = min(m, n)
            fx[:] = 0
            fx[:k] = xx[:k] * xx[:k]
            fx[1:k] += 0.5 * xx[: k - 1]

        Jb = pkg.BandedMatrix(m, n, l, u, device=dev)
        Jb.data.fill_(float("nan"))
        cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device=dev),
                                  torch.zeros(m, dtype=torch.float64, device=dev), "forward", colorvec=cv, sparsity=Jb)
        with fdb_env(SM_COUNT=sm_count):
            pkg.finite_difference_jacobian_(Jb, f_t, x, cache)
        ref = np.full((l + u + 1) * n, np.nan)
        oracle.jacobian(oracle.Problem.banded(m, n, l, u), ref, f_n, xh.copy(), colorvec=cv,
                        eps_override=cache._last_plan.eps())
        assert_same_bits(Jb.data.cpu().numpy(), ref, allow_nan=False)


WIDE_BANDS = [(3000, 3000, 64, 64), (2500, 3100, 70, 58), (3100, 2500, 40, 88), (900, 900, 33, 31)]


@pytest.mark.parametrize("m,n,l,u", WIDE_BANDS)
def test_wide_band_few_colors_with_colourless_columns(pkg, oracle, dev, m, n, l, u):
    # few colours on a wide band: quotients pre-divided in place + whole-band copy; columns without a valid colour stay 0
    # (fill_matrix!), corner slots outside the matrix 0; square / wide / tall, even and odd l+u+1
    _wide_band_case(pkg, oracle, dev, m, n, l, u)


@pytest.mark.parametrize("sm_count", [1, 3])
@pytest.mark.parametrize("m,n,l,u", WIDE_BANDS)
def test_wide_band_multiwave(pkg, oracle, dev, m, n, l, u, sm_count):
    _wide_band_case(pkg, oracle, dev, m, n, l, u, sm_count)


def _wide_band_case(pkg, oracle, dev, m, n, l, u, sm_count=None):
    rng = np.random.default_rng(5)
    cv = cyc_colors(n, 5)
    cv[rng.integers(0, n, 25)] = 0
    x = dev_x(pkg, dev, n, 78)
    xh = oracle.fill_x(n, 78)

    def f_t(fx, xx):
        k = min(m, n)
        fx.zero_()
        fx[:k] = xx[:k] * xx[:k]
        fx[1:k] += 0.5 * xx[: k - 1]

    def f_n(fx, xx):
        k = min(m, n)
        fx[:] = 0
        fx[:k] = xx[:k] * xx[:k]
        fx[1:k] += 0.5 * xx[: k - 1]

    for fdtype in ("forward", "central"):
        Jb = pkg.BandedMatrix(m, n, l, u, device=dev)
        Jb.data.fill_(float("nan"))
        cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device=dev),
                                  torch.zeros(m, dtype=torch.float64, device=dev), fdtype, colorvec=cv, sparsity=Jb)
        with fdb_env(SM_COUNT=sm_count):
            pkg.finite_difference_jacobian_(Jb, f_t, x, cache)
        ref = np.full((l + u + 1) * n, np.nan)
        oracle.jacobian(oracle.Problem.banded(m, n, l, u), ref, f_n, xh.copy(), fdtype=FD[fdtype], colorvec=cv,
                        eps_override=cache._last_plan.eps())
        assert_same_bits(Jb.data.cpu().numpy(), ref, allow_nan=False)


def ell_problem(n, K, C, seed):
    """SURVEY.md §8d config C4 generator (reduced n): row i picks K distinct colours and, per colour, a random column
    of that colour; cyclic colouring -> valid by construction."""
    rng = np.random.default_rng(seed)
    cols = np.empty((n, K), np.int64)
    per_color = n // C
    for i0 in range(0, n, 65536):
        i1 = min(n, i0 + 65536)
        colors = np.argsort(rng.random((i1 - i0, C)), axis=1)[:, :K]
        which = rng.integers(0, per_color, size=(i1 - i0, K))
        cols[i0:i1] = which * C + colors
    coef = rng.uniform(-1, 1, size=(n, K))
    return cols.astype(np.int32), coef


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("strategy", [1, 2, 3])
def test_c4_random_sparse_64_colors_bitexact(pkg, oracle, dev, fdtype, strategy):
    """BASELINE config C4 shape at reduced n: random sparse f!, 8 nnz/row, 64 colours, CSC J — through BOTH scatter
    strategies: 1 = one fused pass over nzval, 2 = per-colour column lists launched after each colour's f!."""
    import scipy.sparse as sps
    n, K, Cc = 64 * 400, 8, 64
    cols, coef = ell_problem(n, K, Cc, 11)
    A = sps.csc_matrix((np.ones(n * K), (np.repeat(np.arange(n), K), cols.reshape(-1))), shape=(n, n))
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    cv = cyc_colors(n, Cc)
    x = dev_x(pkg, dev, n, 0x5EED + 4)
    xh = oracle.fill_x(n, 0x5EED + 4)
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(coef.T)     # ELL layout [K][m]
    d_cols = torch.from_numpy(colsT).to(dev)
    d_coef = torch.from_numpy(coefT).to(dev)
    ctx = pkg._lib.EllCtx(n, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
    J = pkg.SparseMatrixCSC(n, n, t64(colptr), t64(rowval), torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J, strategy=strategy)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_ellrows", ctx), x, cache)
    eps = cache._last_plan.eps()
    info = cache._last_plan.info()
    assert info["strategy"] == (0 if strategy == 1 else 1) and info["mean_row_jump"] > 64
    octx = oracle.SynthEllCtx(n, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    ref = np.full(A.nnz, np.nan)
    r = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_ellrows"), xh.copy(),
                        fdtype=FD[fdtype], colorvec=cv, eps_override=eps, ctx=octx)
    own = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), np.zeros(A.nnz), oracle.native_fn("synth_ellrows"),
                          xh.copy(), fdtype=FD[fdtype], colorvec=cv, ctx=octx)
    assert ctx.calls == r["fcalls"] == (65 if fdtype == "forward" else 128)
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-14)
    assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)
    assert cache._last_plan.info()["color_bits"] == 8


@pytest.mark.parametrize("ncolors,bits", [(300, 16), (70000, 32)])
def test_wide_color_types(pkg, oracle, dev, ncolors, bits):
    # uint16 / int32 colour streams and the windowed eps reduction (C > 512): diagonal + sub-diagonal pattern
    import scipy.sparse as sps
    n = ncolors
    A = sps.diags([np.ones(n - 1), np.ones(n)], [-1, 0], format="csc")
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    cv = np.arange(1, n + 1, dtype=np.int64)
    x = dev_x(pkg, dev, n, 5)
    xh = oracle.fill_x(n, 5)
    J = pkg.SparseMatrixCSC(n, n, t64(colptr), t64(rowval), torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
    ctx = pkg._lib.TridiagCtx(n, 0)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J, max_batch=64)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_tridiag", ctx, 64), x, cache)
    eps = cache._last_plan.eps()
    assert cache._last_plan.info()["color_bits"] == bits
    # per-colour eps = max(relstep*sqrt(|x_k|), absstep): one column per colour
    rel = np.sqrt(np.finfo(float).eps)
    np.testing.assert_allclose(eps, np.maximum(rel * np.sqrt(np.abs(xh)), rel), rtol=1e-14)
    if n <= 1000:
        ref = np.full(A.nnz, np.nan)
        oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_tridiag"), xh.copy(),
                        colorvec=cv, eps_override=eps, ctx=oracle.SynthTridiagCtx(n, 1))
        assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)
    else:
        got = J.to_dense() if n <= 2000 else None
        nz = J.nzval.cpu().numpy()
        assert ctx.calls == n + 1
        # f is the tridiagonal stencil: d f_i/d x_i = -2, d f_{i+1}/d x_i = 1
        col_of = np.repeat(np.arange(1, n + 1), np.diff(colptr))
        np.testing.assert_allclose(nz, np.where(rowval == col_of, -2.0, 1.0), atol=1e-6)


def test_invalid_and_empty_colours(pkg, oracle, dev):
    # colour 0 (never matched: entries stay 0, fill_matrix!), an unused colour (still costs an f! call, jacobians.jl:547)
    N = 12
    colptr, rowval = tridiag_csc(N)
    cv = np.array([1, 2, 4, 0, 2, 4, 1, 2, 4, 1, 0, 4], dtype=np.int64)
    x = dev_x(pkg, dev, N, 9)
    xh = oracle.fill_x(N, 9)
    for fdtype in ("forward", "central"):
        J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
        ctx = pkg._lib.TridiagCtx(N, 0)
        for strategy in (1, 2):
            J.nzval.fill_(float("nan"))
            ctx.calls = 0
            cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J, strategy=strategy)
            pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_tridiag", ctx), x, cache)
            ref = np.full(len(rowval), np.nan)
            r = oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"), xh.copy(),
                                fdtype=FD[fdtype], colorvec=cv, eps_override=cache._last_plan.eps(), ctx=oracle.SynthTridiagCtx(N, 1))
            assert ctx.calls == r["fcalls"] == (5 if fdtype == "forward" else 8)
            assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)


def test_different_pattern_csc_J(pkg, oracle, dev):
    # J::CSC whose pattern is a superset of the sparsity's: generic J[r,c]= path (ext/..SparseArraysExt.jl:20-28);
    # a J lacking a sparsity entry would need insertion -> rejected loudly
    import scipy.sparse as sps
    N = 40
    colptr, rowval = tridiag_csc(N)
    sp = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), None)
    Afull = sps.diags([np.ones(N - 2), np.ones(N - 1), np.ones(N), np.ones(N - 1)], [-2, -1, 0, 1], format="csc")
    J = pkg.SparseMatrixCSC.from_scipy(Afull, dev)
    J.nzval.fill_(float("nan"))
    x = dev_x(pkg, dev, N, 3)
    cache = pkg.JacobianCache(x, "forward", colorvec=cyc_colors(N, 3), sparsity=sp)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_tridiag", pkg._lib.TridiagCtx(N, 0)), x, cache)
    dense = J.to_dense()
    ref = np.zeros(N * N)
    oracle.jacobian(oracle.Problem.csc_to_dense(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"),
                    oracle.fill_x(N, 3), colorvec=cyc_colors(N, 3), eps_override=cache._last_plan.eps(),
                    ctx=oracle.SynthTridiagCtx(N, 1))
    assert_same_bits(dense, ref.reshape(N, N, order="F"), allow_nan=False)
    Jsub = pkg.SparseMatrixCSC.from_scipy(sps.eye(N, format="csc"), dev)
    with pytest.raises(pkg._lib.FdbError) as ei:
        pkg.finite_difference_jacobian_(Jsub, native(pkg, "fdbs_tridiag", pkg._lib.TridiagCtx(N, 0)), x,
                                        pkg.JacobianCache(x, "forward", colorvec=cyc_colors(N, 3), sparsity=sp))
    assert ei.value.status == pkg._lib.FDB_ERR_UNSUPPORTED
    # J's own column pointer is searched by the plan: a decreasing one is rejected, not read out of bounds
    bad = pkg.SparseMatrixCSC.from_scipy(Afull, dev)
    bad.colptr[N // 2] = bad.colptr[N // 2 + 1] + 3
    with pytest.raises(pkg._lib.FdbError) as ei:
        pkg.finite_difference_jacobian_(bad, native(pkg, "fdbs_tridiag", pkg._lib.TridiagCtx(N, 0)), x,
                                        pkg.JacobianCache(x, "forward", colorvec=cyc_colors(N, 3), sparsity=sp))
    assert ei.value.status == pkg._lib.FDB_ERR_INVALID


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("batch", [1, 7])
@pytest.mark.parametrize("n", [300, 301])
def test_dense_columns_bitexact(pkg, oracle, dev, fdtype, batch, n):
    """sparsity === nothing: dense column branch (jacobians.jl:548-557, :590-598), BASELINE config C5 shape at reduced n
    (even n: 16-byte row pairs; odd n: columns are only 8-byte aligned -> scalar rows)."""
    _dense_columns_case(pkg, oracle, dev, fdtype, batch, n)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("batch", [1, 7])
@pytest.mark.parametrize("n,sm_count", [(300, 1), (301, 3), (2049, 1), (2050, 3)])
def test_dense_columns_multiwave(pkg, oracle, dev, fdtype, batch, n, sm_count):
    # the same branch with several grid-stride steps per block (n = 2049: 1024 row pairs per column)
    _dense_columns_case(pkg, oracle, dev, fdtype, batch, n, sm_count)


def _dense_columns_case(pkg, oracle, dev, fdtype, batch, n, sm_count=None):
    w = np.random.default_rng(2).random(n)
    d_w = torch.from_numpy(w).to(dev)
    nblk = (n + 1023) // 1024
    bs = torch.zeros(nblk * max(batch, 1), dtype=torch.float64, device=dev)
    ctx = pkg._lib.Rank1Ctx(n, d_w.data_ptr(), bs.data_ptr(), max(batch, 1), 0)
    x = dev_x(pkg, dev, n, 0x5EED + 5)
    xh = oracle.fill_x(n, 0x5EED + 5)
    J = pkg.zeros_colmajor(n, n, dev)
    J.fill_(float("nan"))
    cache = pkg.JacobianCache(x, fdtype, max_batch=batch)
    with fdb_env(SM_COUNT=sm_count):
        pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_rank1", ctx, batch), x, cache)
    eps = cache._last_plan.eps()
    ref = np.zeros(n * n)
    r = oracle.jacobian(oracle.Problem.dense(n, n), ref, oracle.native_fn("synth_rank1"), xh.copy(), fdtype=FD[fdtype],
                        ctx=oracle.SynthRank1Ctx(n, w.ctypes.data_as(C.POINTER(C.c_double)), 1))
    assert ctx.calls == r["fcalls"] == (n + 1 if fdtype == "forward" else 2 * n)
    assert_same_bits(eps, r["eps"], allow_nan=False)                # per-component step: no reduction involved -> exact
    assert_same_bits(J.cpu().numpy().reshape(-1, order="F"), ref, allow_nan=False)
    analytic = np.diag(2 * xh) + np.outer(w, np.ones(n)) / n
    assert np.max(np.abs(J.cpu().numpy() - analytic)) < (1e-6 if fdtype == "forward" else 1e-8)


def test_host_buffer_entry_point(pkg, oracle, dev):
    # fdb_jacobian_host: HOST x and J storage (pinned), H2D/D2H inside the call
    N = 3000
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), None)
    plan = pkg.make_plan(J, J, cv, "forward", N, dev)
    xh = pkg.pinned_empty(N)
    xh[:] = oracle.fill_x(N, 21)
    Jh = pkg.pinned_empty(len(rowval))
    Jh[:] = np.nan
    fxh = np.zeros(N)
    ctx = pkg._lib.TridiagCtx(N, 0)
    L = pkg._lib
    L.check(L.lib().fdb_jacobian_host(plan.handle, C.cast(L.synth().fdbs_tridiag, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p),
                                      xh.ctypes.data, Jh.ctypes.data, fxh.ctypes.data, None, float("nan"), float("nan"), 1.0))
    ref = np.full(len(rowval), np.nan)
    r = oracle.jacobian(oracle.Problem.csc_same(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"), np.array(xh),
                        colorvec=cv, eps_override=plan.eps(), ctx=oracle.SynthTridiagCtx(N, 1))
    assert_same_bits(Jh, ref, allow_nan=False)
    assert ctx.calls == 4
    assert_same_bits(fxh, r["cache"]["fx"], allow_nan=False)          # cache.fx = f(x) in forward mode (jacobians.jl:541)


def test_error_paths(pkg, dev):
    L = pkg._lib
    N = 10
    colptr, rowval = tridiag_csc(N)
    x = dev_x(pkg, dev, N, 1)
    J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.zeros(len(rowval), dtype=torch.float64, device=dev))
    # callback failure aborts and is surfaced
    with pytest.raises(L.FdbError) as ei:
        pkg.finite_difference_jacobian_(J, pkg.NativeFn(C.cast(L.synth().fdbs_fail, C.c_void_p).value, None), x,
                                        pkg.JacobianCache(x, "forward", colorvec=cyc_colors(N, 3), sparsity=J))
    assert ei.value.status == L.FDB_ERR_CALLBACK
    # broken colptr
    bad = colptr.copy()
    bad[3] = bad[2] - 1
    with pytest.raises(L.FdbError) as ei:
        pkg.make_plan(J, pkg.SparseMatrixCSC(N, N, t64(bad), t64(rowval), None), None, "forward", N, dev)
    assert ei.value.status == L.FDB_ERR_INVALID
    # row index out of range
    badr = rowval.copy()
    badr[5] = N + 3
    with pytest.raises(L.FdbError):
        pkg.make_plan(J, pkg.SparseMatrixCSC(N, N, t64(colptr), t64(badr), None), None, "forward", N, dev)
    # unknown fdtype (epsilons.jl:159-167)
    with pytest.raises(ValueError, match="Unrecognized fdtype"):
        pkg.JacobianCache(x, "hcentral")
    # row-major dense J is not a Julia Matrix
    with pytest.raises(ValueError, match="column-major"):
        pkg.finite_difference_jacobian_(torch.zeros(N, N, dtype=torch.float64, device=dev), lambda a, b: None, x, "forward")
    # CPU tensors are rejected loudly — no CPU fallback
    with pytest.raises(TypeError):
        pkg.JacobianCache(torch.zeros(3, dtype=torch.float64), "forward")


def test_resize(pkg, dev):
    # resize!(cache, i) jacobians.jl:655-661
    x = torch.rand(4, dtype=torch.float64, device=dev)
    c = pkg.JacobianCache(x, "forward")
    pkg.resize_(c, 6)
    assert c.x1.numel() == 6 and c.fx.numel() == 6 and c.fx1.numel() == 6 and c.colorvec == range(1, 7)
    x6 = torch.rand(6, dtype=torch.float64, device=dev)
    J = pkg.zeros_colmajor(6, 6, dev)
    pkg.finite_difference_jacobian_(J, lambda fx, xx: fx.copy_(xx * xx), x6, c)
    np.testing.assert_allclose(J.cpu().numpy(), np.diag(2 * x6.cpu().numpy()), atol=1e-6)


@pytest.mark.parametrize("kind", ["mod12", "mod20", "mod40", "random50", "random50_with_invalid"])
def test_window_eps_lane_groups(pkg, oracle, dev, kind):
    # C > 8 takes the shared-memory window reduction; the plan picks the widest conflict-free lane group
    # (8 / 16 / 32 for cyclic colourings) or the match.any fallback (arbitrary colourings).  eps must agree with the
    # reference formula (jacobians.jl:559-561) and J must be bit-identical to the oracle run with the device's eps.
    n = 5003
    colptr, rowval = tridiag_csc(n)
    rng = np.random.default_rng(7)
    if kind.startswith("mod"):
        cv = (np.arange(n, dtype=np.int64) % int(kind[3:])) + 1
    else:
        cv = rng.integers(1, 51, n).astype(np.int64)
        if kind.endswith("invalid"):
            cv[rng.integers(0, n, 40)] = 0
    x = dev_x(pkg, dev, n, 9)
    xh = oracle.fill_x(n, 9)
    J = pkg.SparseMatrixCSC(n, n, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
    ctx = pkg._lib.TridiagCtx(n, 0)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J, max_batch=16)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_tridiag", ctx, 16), x, cache)
    eps = cache._last_plan.eps()
    C = int(cv.max())
    rel = np.sqrt(np.finfo(float).eps)
    ss = np.array([np.sum(xh[cv == k] ** 2) for k in range(1, C + 1)])
    np.testing.assert_allclose(eps, np.maximum(rel * np.sqrt(np.sqrt(ss)), rel), rtol=1e-13)
    ref = np.full(len(rowval), np.nan)
    oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_tridiag"), xh.copy(),
                    colorvec=cv, eps_override=eps, ctx=oracle.SynthTridiagCtx(n, 1))
    assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_kat_identity_map_all_fdtypes(pkg, golden, dev, fdtype):
    # finitedifftests.jl:600-605: in-place Jacobian of the identity map at ones(2), every fdtype: J ≈ I; the caller's x is
    # untouched (the cache-less entry builds exactly this cache: api.finite_difference_jacobian_, jacobians.jl:456-467)
    g = golden["identity2"]
    x = torch.tensor(g["x"], dtype=torch.float64, device=dev)

    def ident(out, xx):
        out.copy_(xx)

    J = pkg.zeros_colmajor(2, 2, dev)
    J.fill_(float("nan"))
    pkg.finite_difference_jacobian_(J, ident, x, pkg.JacobianCache(x, fdtype))
    np.testing.assert_allclose(J.cpu().numpy(), np.array(g["J_expected"]), rtol=g["rtol"], atol=g["rtol"])
    assert_same_bits(x.cpu(), torch.tensor(g["x"], dtype=torch.float64), allow_nan=False)
