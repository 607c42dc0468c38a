"""Randomised GPU-vs-oracle parity (bit-exact): random CSC patterns (ragged columns, empty columns, supersets of the
function's true dependence), random — not necessarily valid — colourings (shared rows inside a colour must reproduce the
reference's "spurious" values, invalid colours must stay zero), m != n, forward / central / complex-free, f_in, dir,
drift on/off, every scatter strategy (storage-order pass, colour-major lists per group / in one launch), small scratch
budgets (several groups per Jacobian), batched callbacks, dense-J destinations."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sps

from _util import assert_same_bits, fdb_env

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


def _case(rng, pkg, oracle, dev, sm_count=None, lo=1, hi=400):
    L = pkg._lib
    m = int(rng.integers(lo, hi))
    n = int(rng.integers(lo, hi))
    K = int(rng.integers(1, 6))
    cols = rng.integers(0, n, size=(m, K)).astype(np.int32)          # random dependence, duplicates allowed
    coef = rng.uniform(-1, 1, size=(m, K))
    # J pattern: the true dependence plus random extra structural entries (their values must come out as computed)
    extra = int(rng.integers(0, m + 1))
    er, ec = rng.integers(0, m, extra), rng.integers(0, n, extra)
    A = sps.csc_matrix((np.ones(m * K + extra), (np.concatenate([np.repeat(np.arange(m), K), er]),
                                                 np.concatenate([cols.reshape(-1), ec]))), shape=(m, n))
    A.sum_duplicates()
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    ncol = int(rng.integers(1, 12))
    cv = rng.integers(0 if rng.random() < 0.3 else 1, ncol + 1, size=n).astype(np.int64)   # 0 = no valid colour
    if cv.max() < 1:
        cv[0] = 1
    fdtype = "forward" if rng.random() < 0.5 else "central"
    opts = dict(no_drift=bool(rng.random() < 0.3), strategy=int(rng.integers(0, 4)), max_batch=int(rng.integers(1, 4)))
    if rng.random() < 0.35:
        # a scratch budget of a few slabs: several scatter groups per Jacobian (colour-major lists: one launch per group,
        # f(x) pre-gathered into list order; storage-order pass: ownership tests per group)
        opts["scratch_bytes"] = int(8 * (m + 2) * (2 if fdtype == "central" else 1) * int(rng.integers(1, 4)) + 64)
    dense_J = rng.random() < 0.3 and m * n <= 4_000_000
    x = torch.from_numpy(rng.uniform(-2, 2, n)).to(dev)
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(coef.T)
    d_cols, d_coef = torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev)
    ctx = L.EllCtx(m, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx, max_batch=opts["max_batch"])
    sp = pkg.SparseMatrixCSC(m, n, torch.from_numpy(colptr), torch.from_numpy(rowval),
                             torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
    fx = torch.zeros(m, dtype=torch.float64, device=dev)
    cache = pkg.JacobianCache(x.clone(), fx, fx.clone(), fdtype, colorvec=cv, sparsity=sp, **opts)
    octx = oracle.SynthEllCtx(m, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    kw = {}
    use_fin = fdtype == "forward" and rng.random() < 0.3
    dirv = -1.0 if (fdtype == "forward" and rng.random() < 0.3) else 1.0
    fin_t = None
    if use_fin:
        fin = np.zeros(m)
        oracle.lib().synth_ellrows(C.byref(octx), fin.ctypes.data_as(C.POINTER(C.c_double)),
                                   x.cpu().numpy().ctypes.data_as(C.POINTER(C.c_double)))
        fin_t = torch.from_numpy(fin).to(dev)
        kw["f_in"] = fin
    if dense_J:
        J = pkg.zeros_colmajor(m, n, dev)
        J.fill_(float("nan"))
        P = oracle.Problem.csc_to_dense(m, n, colptr, rowval)
        ref = np.full(m * n, np.nan)
    else:
        J = sp
        P = oracle.Problem.csc_same(m, n, colptr, rowval)
        ref = np.full(A.nnz, np.nan)
    with fdb_env(SM_COUNT=sm_count):       # grids sized as if the device had sm_count SMs: several tiles per block
        pkg.finite_difference_jacobian_(J, f, x, cache, fin_t, dir=dirv)
        torch.cuda.synchronize()
    eps = cache._last_plan.eps()
    r = oracle.jacobian(P, ref, oracle.native_fn("synth_ellrows"), x.cpu().numpy().copy(), fdtype=0 if fdtype == "forward" else 1,
                        colorvec=cv, eps_override=eps, no_drift=opts["no_drift"], dir=dirv, ctx=octx, **kw)
    got = (J.cpu().numpy().reshape(-1, order="F") if dense_J else sp.nzval.cpu().numpy())
    desc = f"m={m} n={n} K={K} C={cv.max()} {fdtype} {opts} dense={dense_J} f_in={use_fin} dir={dirv} sm_count={sm_count}"
    assert ctx.calls == r["fcalls"], desc
    assert_same_bits(got, ref, desc)
    own = oracle.jacobian(P, np.zeros_like(ref), oracle.native_fn("synth_ellrows"), x.cpu().numpy().copy(),
                          fdtype=0 if fdtype == "forward" else 1, colorvec=cv, dir=dirv, ctx=octx, **kw)
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-13, err_msg=desc)


def test_random_patterns_bitexact(pkg, oracle):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(20260924)
    for _ in range(120):
        _case(rng, pkg, oracle, dev)


@pytest.mark.parametrize("sm_count", [1, 3])
def test_random_patterns_bitexact_multiwave(pkg, oracle, sm_count):
    # the same generator with the grids sized as if the device had sm_count SMs
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(20260924)
    for _ in range(60):
        _case(rng, pkg, oracle, dev, sm_count)


@pytest.mark.parametrize("sm_count", [1, 3])
def test_random_patterns_mid_size_multiwave(pkg, oracle, sm_count):
    # m, n of 10^4 .. 10^5 under FDB_SM_COUNT: every scatter form, the perturbation and step-size passes several tiles
    # per block
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(20261015 + sm_count)
    for _ in range(8):
        _case(rng, pkg, oracle, dev, sm_count, lo=10_000, hi=100_000)
