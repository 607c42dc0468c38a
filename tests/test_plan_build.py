"""Plan construction through the C ABI (run with -m gpu).

Every rejection path of every creator returns its status, leaves the output handle NULL and names the cause in
fdb_last_error().  A plan keeps only the device memory a Jacobian call reads: the scratch used while it is built (the
error flag, colour counters, the 32-bit column stream of a dense-J plan, the staged form's row offsets when that form
is rejected) is freed before the creator returns, so device_bytes does not count it.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import fdb_env  # noqa: E402


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()._lib


SENTINEL = 0x1234


def i64(*v):
    return np.array(v, dtype=np.int64)


def ptr(a):
    return None if a is None else a.ctypes.data


def _opts(L, fdtype=0):
    o = L.PlanOpts()
    o.fdtype = fdtype
    o.use_current_device = 1
    return o


def _rejects(L, create, status, cause):
    """create(handle_ref) must fail with `status`, leave the handle NULL and name `cause` in fdb_last_error()."""
    h = C.c_void_p(SENTINEL)
    st = create(C.byref(h))
    err = L.lib().fdb_last_error().decode()
    if st == L.FDB_OK and h.value:
        L.lib().fdb_plan_destroy(h)
    assert st == status, f"status {st}, expected {status}: {err}"
    assert h.value is None, "handle not NULL after a failed create"
    assert cause in err, f"{cause!r} not in {err!r}"


# 4x4 diagonal pattern, 1-based CSC as SparseMatrixCSC stores it
DIAG_CP, DIAG_RV = i64(1, 2, 3, 4, 5), i64(1, 2, 3, 4)


def _csc(L, *, colptr=DIAG_CP, rowval=DIAG_RV, jkind=0, j_colptr=None, j_rowval=None, ldJ=0, m=4, n=4):
    o = _opts(L)
    return lambda h: L.lib().fdb_plan_create_csc(h, m, n, ptr(colptr), ptr(rowval), jkind, ptr(j_colptr), ptr(j_rowval),
                                                 ldJ, None, C.byref(o))


CSC_CASES = {
    "null_colptr": (dict(colptr=None), "INVALID", "colptr is NULL"),
    "bad_jkind": (dict(jkind=2), "INVALID", "CSC sparsity supports J kinds"),
    "colptr_end_out_of_range": (dict(colptr=i64(1, 2, 3, 4, 0)), "UNSUPPORTED", "nnz=-1 unsupported"),
    "null_rowval": (dict(rowval=None), "INVALID", "rowval is NULL"),
    "bad_J_colptr": (dict(j_colptr=i64(1, 2, 3, 4, 0), j_rowval=i64(1, 2, 3, 4)), "INVALID",
                     "J.colptr[n+1]=0 is not a valid CSC end pointer"),
    "ldJ_below_m": (dict(jkind=1, ldJ=3), "INVALID", "ldJ=3 < m=4"),
    "row_out_of_range": (dict(rowval=i64(1, 2, 5, 4)), "INVALID", "row index outside 1..m"),
    "entry_missing_from_J": (dict(j_colptr=i64(1, 2, 3, 4, 5), j_rowval=i64(2, 2, 3, 4)), "UNSUPPORTED",
                             "absent from J's CSC pattern"),
}


@pytest.mark.parametrize("case", sorted(CSC_CASES))
def test_csc_rejections(L, case):
    kw, status, cause = CSC_CASES[case]
    _rejects(L, _csc(L, **kw), getattr(L, f"FDB_ERR_{status}"), cause)


def _coo(L, *, rows=i64(1, 2, 3, 4), cols=i64(1, 2, 3, 4), jkind=3, slots=i64(1, 2, 3, 4), ld=4):
    o = _opts(L)
    return lambda h: L.lib().fdb_plan_create_coo(h, 4, 4, 4, ptr(rows), ptr(cols), jkind, ptr(slots), ld, None, C.byref(o))


COO_CASES = {
    "null_indices": (dict(rows=None), "rows_index/cols_index NULL"),
    "bad_jkind": (dict(jkind=0), "COO sparsity supports J kinds DENSE and SLOTS"),
    "null_slots": (dict(slots=None), "slots is NULL"),
    "ldJ_below_m": (dict(jkind=1, ld=3), "ldJ < m"),
}


@pytest.mark.parametrize("case", sorted(COO_CASES))
def test_coo_rejections(L, case):
    kw, cause = COO_CASES[case]
    _rejects(L, _coo(L, **kw), L.FDB_ERR_INVALID, cause)


@pytest.mark.parametrize("jkind,l,u,cause", [(0, 1, 1, "banded sparsity supports J kinds BAND and DENSE"),
                                             (2, -2, 0, "invalid bandwidths l=-2 u=0")])
def test_banded_rejections(L, jkind, l, u, cause):
    o = _opts(L)
    _rejects(L, lambda h: L.lib().fdb_plan_create_banded(h, 4, 4, l, u, jkind, 4, None, C.byref(o)), L.FDB_ERR_INVALID,
             cause)


def test_dense_rejections(L):
    o = _opts(L)
    _rejects(L, lambda h: L.lib().fdb_plan_create_dense(h, 4, 4, 3, C.byref(o)), L.FDB_ERR_INVALID, "ldJ < m")
    cv = i64(1, 2, 5, 1)
    _rejects(L, lambda h: L.lib().fdb_plan_create_dense_colorvec(h, 4, 4, 4, ptr(cv), C.byref(o)), L.FDB_ERR_INVALID,
             "maximum(colorvec)=5 indexes x beyond length(x)=4")


def test_jvp_rejects_complex(L):
    o = _opts(L, fdtype=L.FDB_COMPLEX)
    _rejects(L, lambda h: L.lib().fdb_jvp_plan_create(h, 4, 4, C.byref(o)), L.FDB_ERR_UNSUPPORTED,
             "doesn't support :complex-mode")


def test_group_rejects_device_out_of_range(L):
    count = L.lib().fdb_device_count()
    devs = (C.c_int * 2)(0, count)
    _rejects(L, lambda h: L.lib().fdb_group_create_dense(h, 2, devs, 4, 4, 4, None), L.FDB_ERR_INVALID,
             f"device {count} out of range")


def _random_csc(m, n, per_col, seed):
    """CSC pattern with `per_col` distinct random rows per column: its rows jump all over, so it is not row-local."""
    rng = np.random.default_rng(seed)
    rows = np.sort(np.stack([rng.choice(m, per_col, replace=False) for _ in range(n)]), axis=1)
    colptr = (1 + per_col * np.arange(n + 1)).astype(np.int64)
    return colptr, (rows.reshape(-1) + 1).astype(np.int64)


def _device_bytes(L, m, n, colptr, rowval, colorvec, jkind=0):
    o = _opts(L)
    h = C.c_void_p()
    L.check(L.lib().fdb_plan_create_csc(C.byref(h), m, n, ptr(colptr), ptr(rowval), jkind, None, None,
                                        m if jkind == 1 else 0, ptr(colorvec), C.byref(o)))
    try:
        info = L.PlanInfo()
        L.check(L.lib().fdb_plan_info(h, C.byref(info)))
        return info
    finally:
        L.lib().fdb_plan_destroy(h)


def test_rejected_staged_form_is_not_kept(L):
    """<= 7 colours, nzval J, one GPU: the plan builds the staged form's row offsets, then rejects the form because the
    pattern is not row-local.  It must hold exactly what the same plan holds when the staged form is never tried."""
    m = n = 20000
    colptr, rowval = _random_csc(m, n, 4, seed=3)
    colorvec = (np.arange(n) % 7 + 1).astype(np.int64)
    with fdb_env(NO_STAGED=None):
        tried = _device_bytes(L, m, n, colptr, rowval, colorvec)
    with fdb_env(NO_STAGED=1):
        skipped = _device_bytes(L, m, n, colptr, rowval, colorvec)
    assert tried.staged == 0 and tried.strategy == 0 and tried.n_groups == 1
    assert len(rowval) >= 1024
    assert tried.device_bytes == skipped.device_bytes


def test_dense_J_keeps_only_its_destination_stream(L):
    """8..15 colours (no staged form, no colour-major lists): a dense-J plan holds the nzval plan's memory plus its
    8-byte destination per entry, and not the 32-bit column stream it is built from."""
    m = n = 20000
    colptr, rowval = _random_csc(m, n, 4, seed=5)
    colorvec = (np.arange(n) % 12 + 1).astype(np.int64)
    nz = _device_bytes(L, m, n, colptr, rowval, colorvec, jkind=L.FDB_J_CSC_NZVAL)
    dense = _device_bytes(L, m, n, colptr, rowval, colorvec, jkind=L.FDB_J_DENSE)
    assert nz.strategy == 0 and dense.strategy == 0 and nz.staged == 0
    assert dense.device_bytes - nz.device_bytes == 8 * len(rowval)
