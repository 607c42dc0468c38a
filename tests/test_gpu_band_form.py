"""Band form of the staged scatter and the cyclic colour source, bit for bit.

A CSC pattern that is exactly a clipped band (column c holds rows max(0, c-l) .. min(m-1, c+u), in order) makes the staged
diff+scatter pass derive every entry's row and column from its position instead of reading the 16-bit row offsets; a
colouring with colorvec[j] == j mod P + 1 makes the step-size, perturbation and band scatter kernels compute colours
instead of reading them.  Every case is compared bit for bit with the oracle (fed the device step sizes) and with the
same plan built under FDB_NO_BAND=1 (indexed form); the path a plan took is read from moved_bytes_scatter:
band form 8*E + 8*m*(windows) (+ n colour bytes unless the colouring is cyclic)."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, band_csc, fdb_env

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


def band_rows(m, n, l, u):
    return [list(range(max(0, c - l), min(m - 1, c + u) + 1)) for c in range(n)]


def to_csc(cols):
    colptr = np.cumsum([0] + [len(r) for r in cols]).astype(np.int64) + 1
    rowval = np.array([r for rr in cols for r in rr], dtype=np.int64) + 1
    return colptr, rowval


def cyclic(n, P):
    return (np.arange(n) % P + 1).astype(np.int64)


def run(pkg, oracle, m, n, colptr, rowval, cv, fdtype, seed, no_band=False, f_in=False, dirv=1.0, no_drift=False,
        sm_count=None):
    L = pkg._lib
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(seed)
    K = 3
    cols = rng.integers(0, n, size=(m, K)).astype(np.int32)
    coef = rng.uniform(-1, 1, size=(m, K))
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(coef.T)
    d_cols, d_coef = torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev)
    x = torch.from_numpy(rng.uniform(-2, 2, n)).to(dev)
    E = len(rowval)
    ctx = L.EllCtx(m, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx)
    sp = pkg.SparseMatrixCSC(m, n, torch.from_numpy(colptr), torch.from_numpy(rowval),
                             torch.full((E,), float("nan"), dtype=torch.float64, device=dev))
    octx = oracle.SynthEllCtx(m, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    kw, fin_t = {}, None
    if f_in:
        fin = np.zeros(m)
        oracle.lib().synth_ellrows(C.byref(octx), fin.ctypes.data_as(C.POINTER(C.c_double)),
                                   x.cpu().numpy().ctypes.data_as(C.POINTER(C.c_double)))
        fin_t = torch.from_numpy(fin).to(dev)
        kw["f_in"] = fin
    with fdb_env(NO_BAND=1 if no_band else None, SM_COUNT=sm_count):
        fx = torch.zeros(m, dtype=torch.float64, device=dev)
        cache = pkg.JacobianCache(x.clone(), fx, fx.clone(), fdtype, colorvec=cv, sparsity=sp, no_drift=no_drift)
        pkg.finite_difference_jacobian_(sp, f, x, cache, fin_t, dir=dirv)
        torch.cuda.synchronize()
    plan = cache._last_plan
    eps = plan.eps()
    got = sp.nzval.cpu().numpy()
    ref = np.full(E, np.nan)
    r = oracle.jacobian(oracle.Problem.csc_same(m, n, colptr, rowval), ref, oracle.native_fn("synth_ellrows"),
                        x.cpu().numpy().copy(), fdtype=0 if fdtype == "forward" else 1, colorvec=cv, eps_override=eps,
                        no_drift=no_drift, dir=dirv, ctx=octx, **kw)
    assert ctx.calls == r["fcalls"]
    assert_same_bits(got, ref)
    own = oracle.jacobian(oracle.Problem.csc_same(m, n, colptr, rowval), np.zeros(E), oracle.native_fn("synth_ellrows"),
                          x.cpu().numpy().copy(), fdtype=0 if fdtype == "forward" else 1, colorvec=cv, no_drift=no_drift,
                          dir=dirv, ctx=octx, **kw)
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-13)
    return got, eps, plan.info()


def band_bytes(info, m, n, E, C_, fdtype, is_cyclic):
    nwin = 2 * C_ if fdtype == "central" else C_ + 1
    return 8 * E + 8 * m * nwin + (0 if is_cyclic else n * info["color_bits"] // 8)


def check(pkg, oracle, m, n, cols, cv, fdtype, expect_band, is_cyclic=None, seed=1, **kw):
    colptr, rowval = cols if isinstance(cols, tuple) else to_csc(cols)
    E = len(rowval)
    C_ = int(cv.max())
    if is_cyclic is None:
        is_cyclic = bool(np.array_equal(cv, cyclic(n, C_)))
    got, eps, info = run(pkg, oracle, m, n, colptr, rowval, cv, fdtype, seed, **kw)
    got0, eps0, info0 = run(pkg, oracle, m, n, colptr, rowval, cv, fdtype, seed, no_band=True, **kw)
    assert_same_bits(eps, eps0, allow_nan=False)
    assert_same_bits(got, got0)
    want = band_bytes(info, m, n, E, C_, fdtype, is_cyclic)
    if expect_band:
        assert info["staged"] == 1
        assert info["moved_bytes_scatter"] == want, (info["moved_bytes_scatter"], want)
    else:
        assert info["moved_bytes_scatter"] != want
    assert info0["moved_bytes_scatter"] != band_bytes(info0, m, n, E, C_, fdtype, is_cyclic)


FDTYPES = ["forward", "central"]


@pytest.mark.parametrize("fdtype", FDTYPES)
@pytest.mark.parametrize("m,n,l,u", [
    (5000, 5000, 1, 1),       # tridiagonal: E = 14998, not a multiple of 1024
    (3000, 3000, 2, 0),       # l != u (lower band)
    (3000, 3000, 0, 3),       # upper band
    (3000, 1000, 5, 2),       # m > n
    (800, 3000, 1, 4),        # m < n: empty columns after row m
    (4096, 4096, 0, 0),       # diagonal, E a multiple of 1024
    (1200, 1, 0, 1100),       # n = 1
    (700, 2, 0, 600),         # n = 2
    (500, 3, 0, 400),         # n = 3
    (2049, 2049, 1, -1),      # the subdiagonal alone (l = 1, u = -1): column 0 is empty
])
def test_exact_band(pkg, oracle, fdtype, m, n, l, u):
    cols = band_rows(m, n, l, u)
    P = min(n, l + u + 1 if l + u + 1 > 0 else 1, 3 if fdtype == "central" else 6)
    P = max(P, 1)
    # a valid cyclic colouring needs P >= l+u+1; validity does not matter to the bit comparison
    check(pkg, oracle, m, n, cols, cyclic(n, P), fdtype, expect_band=True)


@pytest.mark.parametrize("fdtype", FDTYPES)
def test_below_one_tile(pkg, oracle, fdtype):
    m = n = 300                                   # E = 898 < 1024: not staged at all
    check(pkg, oracle, m, n, band_rows(m, n, 1, 1), cyclic(n, 3), fdtype, expect_band=False)


@pytest.mark.parametrize("fdtype", FDTYPES)
@pytest.mark.parametrize("edit", ["removed", "added"])
def test_near_miss_patterns_fall_back(pkg, oracle, fdtype, edit):
    m = n = 4000
    cols = band_rows(m, n, 1, 1)
    if edit == "removed":
        cols[1777] = [r for r in cols[1777] if r != 1778]
    else:
        cols[2500] = sorted(cols[2500] + [2503])
    check(pkg, oracle, m, n, cols, cyclic(n, 3), fdtype, expect_band=False)


@pytest.mark.parametrize("fdtype", FDTYPES)
@pytest.mark.parametrize("kind", ["cyclic_P4", "off_cycle", "shifted", "colour_0"])
def test_colourings(pkg, oracle, fdtype, kind):
    m = n = 5000
    cols = band_rows(m, n, 1, 1)
    cv = cyclic(n, 3)
    is_cyclic = False
    if kind == "cyclic_P4":                       # P != l+u+1
        cv, is_cyclic = cyclic(n, 4), True
    elif kind == "off_cycle":
        cv[2345] = cv[2345] % 3 + 1
    elif kind == "shifted":
        cv = ((np.arange(n) + 1) % 3 + 1).astype(np.int64)
    else:
        cv[1234] = 0                              # no valid colour: the column's entries stay 0
    check(pkg, oracle, m, n, cols, cv, fdtype, expect_band=True, is_cyclic=is_cyclic)


def test_f_in_dir_no_drift(pkg, oracle):
    m = n = 5000
    cols = band_rows(m, n, 1, 1)
    check(pkg, oracle, m, n, cols, cyclic(n, 3), "forward", expect_band=True, f_in=True)
    check(pkg, oracle, m, n, cols, cyclic(n, 3), "forward", expect_band=True, dirv=-1.0)
    for fdtype in FDTYPES:
        check(pkg, oracle, m, n, cols, cyclic(n, 3), fdtype, expect_band=True, no_drift=True)


@pytest.mark.parametrize("sm_count", [1, 3])
@pytest.mark.parametrize("fdtype,m,n,l,u,colouring", [
    ("forward", 40000, 40000, 2, 1, "cyclic"),     # l != u
    ("central", 40000, 40000, 2, 1, "cyclic"),
    ("forward", 20000, 60000, 1, 4, "cyclic"),     # m < n: empty columns after row m
    ("central", 60000, 30000, 3, 0, "cyclic"),     # m > n
    ("forward", 50000, 50000, 1, 1, "shifted"),    # non-cyclic colouring: the column colour table is read
    ("central", 50000, 50000, 1, 1, "colour_0"),
])
def test_exact_band_multiwave(pkg, oracle, sm_count, fdtype, m, n, l, u, colouring):
    # FDB_SM_COUNT=k sizes the grids as if the device had k SMs: the staged scatter walks several tiles per block
    # (pipeline refill, mbarrier parity flip, reverse walk, the block that takes the partial last tile)
    colptr, rowval = band_csc(m, n, l, u)
    P = min(l + u + 1, 3 if fdtype == "central" else 6)
    cv, is_cyclic = cyclic(n, P), True
    if colouring == "shifted":
        cv, is_cyclic = ((np.arange(n) + 1) % P + 1).astype(np.int64), False
    elif colouring == "colour_0":
        cv[np.arange(17, n, 997)] = 0
        is_cyclic = False
    assert len(rowval) >= 3 * 8 * 3 * 1024      # >= 3 tiles per block at k = 3 with 8 resident blocks per SM
    check(pkg, oracle, m, n, (colptr, rowval), cv, fdtype, expect_band=True, is_cyclic=is_cyclic, sm_count=sm_count)
