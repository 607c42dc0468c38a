"""Shared helpers for the parity tests: pattern builders in the reference's (Julia) conventions —
Int64, 1-based CSC exactly as SparseMatrixCSC stores it."""
import contextlib
import os

import numpy as np
import scipy.sparse as sp


def _host_f64(a):
    if hasattr(a, "detach"):                     # torch tensor, on any device
        a = a.detach().cpu().numpy()
    a = np.asarray(a)
    assert a.dtype == np.float64, f"assert_same_bits compares float64 data, got {a.dtype}"
    return np.ascontiguousarray(a).reshape(-1)


def assert_same_bits(got, ref, what="", *, allow_nan=True):
    """Bit-for-bit equality of two float64 arrays (numpy arrays or torch tensors, CUDA ones included).

    The values are compared as uint64 bit patterns, so +0.0 and -0.0 differ (`==` and np.array_equal treat them as
    equal).  Every NaN counts as one class, whatever its sign and payload: the CPU and the GPU encode the NaNs they
    produce differently.  allow_nan=False also fails on any NaN, as np.array_equal without equal_nan does (for results
    that must be NaN-free, e.g. a J buffer pre-filled with NaN that every slot has to overwrite).  On a mismatch the
    message names the first differing index and both hex patterns."""
    g, r = _host_f64(got), _host_f64(ref)
    assert g.shape == r.shape, f"{what}: shapes differ, {g.shape} vs {r.shape}"
    if not allow_nan:
        assert not (np.isnan(g).any() or np.isnan(r).any()), f"{what}: NaN where none is expected"
    gb, rb = g.view(np.uint64), r.view(np.uint64)
    gn, rn = np.isnan(g), np.isnan(r)
    bad = np.flatnonzero((gb != rb) & ~(gn & rn))
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.size} of {g.size} values differ in their bits; first at index {i}: "
                             f"got {g[i]!r} (0x{int(gb[i]):016x}), expected {r[i]!r} (0x{int(rb[i]):016x})")


@contextlib.contextmanager
def fdb_env(**switches):
    """Set FDB_* switches (DESIGN.md §4) while plans are created, restoring the previous environment afterwards.
    fdb_env(NO_BAND=1, SM_COUNT=3) sets FDB_NO_BAND=1 and FDB_SM_COUNT=3; a value of None leaves the variable unset.
    Plans read the switches once, when they are created (for the Python mirror: on the first call that needs the plan)."""
    names = {f"FDB_{k}": v for k, v in switches.items()}
    saved = {k: os.environ.get(k) for k in names}
    try:
        for k, v in names.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def band_csc(m, n, l, u):
    """colptr/rowval (1-based Int64) of the clipped band: column c holds rows max(0, c-l) .. min(m-1, c+u)."""
    c = np.arange(n)
    lo, hi = np.maximum(c - l, 0), np.minimum(c + u, m - 1)
    cnt = np.maximum(hi - lo + 1, 0)
    colptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    rowval = np.arange(colptr[-1], dtype=np.int64) - np.repeat(colptr[:-1], cnt) + np.repeat(lo, cnt)
    return colptr + 1, rowval + 1


def tridiag_csc(n):
    """colptr/rowval (1-based Int64) of the n x n tridiagonal pattern (sparse(second_derivative_stencil))."""
    A = sp.diags([np.ones(n - 1), np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csc")
    A.sort_indices()
    return (A.indptr.astype(np.int64) + 1), (A.indices.astype(np.int64) + 1)


def csc_from_dense_pattern(A):
    S = sp.csc_matrix(np.asarray(A) != 0)
    S.sort_indices()
    return S.indptr.astype(np.int64) + 1, S.indices.astype(np.int64) + 1


def csc_to_dense(m, n, colptr, rowval, nzval):
    J = np.zeros((m, n))
    for c in range(n):
        for p in range(colptr[c] - 1, colptr[c + 1] - 1):
            J[rowval[p] - 1, c] = nzval[p]
    return J


def band_to_dense(m, n, l, u, data):
    """BandedMatrices storage data[(l+u+1) x n] column-major flat -> dense."""
    w = l + u + 1
    J = np.zeros((m, n))
    for c in range(1, n + 1):
        for r in range(max(1, c - u), min(m, c + l) + 1):
            J[r - 1, c - 1] = data[(c - 1) * w + (u + r - c)]
    return J


def cyc_colors(n, C):
    return (np.arange(n, dtype=np.int64) % C) + 1


def f_tridiag(dx, x):
    # test/coloring_tests.jl:5-13
    n = len(x)
    dx[1:n - 1] = (x[0:n - 2] - 2 * x[1:n - 1]) + x[2:n]
    dx[0] = -2 * x[0] + x[1]
    dx[n - 1] = x[n - 2] - 2 * x[n - 1]


def tridiagonal_coo(n):
    """Structural nz of Julia's Tridiagonal(dl,d,du) as (rows, cols, slots) with slots into [dl; d; du]
    (1-based): band order sub-diagonal, diagonal, super-diagonal."""
    rows = np.concatenate([np.arange(2, n + 1), np.arange(1, n + 1), np.arange(1, n)]).astype(np.int64)
    cols = np.concatenate([np.arange(1, n), np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int64)
    slots = np.arange(1, 3 * n - 1, dtype=np.int64)
    return rows, cols, slots


def tridiagonal_to_dense(n, buf):
    dl, d, du = buf[: n - 1], buf[n - 1: 2 * n - 1], buf[2 * n - 1:]
    return np.diag(d) + np.diag(dl, -1) + np.diag(du, 1)
