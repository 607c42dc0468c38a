"""The CSR plan without a GPU: the mirror type SparseMatrixCSR against scipy, the routing of a CSR J and of a CSR sparsity,
and a Python restatement of diff_scatter_csr's tile and row-search arithmetic (kernels_csr.cuh) checked against scipy's
row of every stored entry on patterns with empty rows, rows longer than a tile, unsorted and repeated columns and tiles
that span thousands of empty rows."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

TILE = 256 * 4          # kCsrTile = kThreads * kCsrPer
STAGE = TILE            # kCsrStage


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


def _csr(rowptr0, cols0, m, n):
    """a scipy CSR holding exactly these stored entries, in this order (no sorting, no summing of duplicates)"""
    A = sp.csr_matrix((np.ones(len(cols0)), np.asarray(cols0, np.int32), np.asarray(rowptr0, np.int32)), shape=(m, n))
    return A


def _patterns():
    rng = np.random.default_rng(7)
    out = {}
    # random with empty rows and unsorted columns
    m, n = 3000, 2500
    lens = rng.integers(0, 6, m)
    lens[rng.random(m) < 0.3] = 0
    rp = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([rng.permutation(n)[:k] for k in lens]) if lens.sum() else np.zeros(0, np.int64)
    out["random_unsorted"] = (rp, cols, m, n)
    # rows longer than a tile, next to short and empty ones
    lens = np.array([0, 3000, 1, 0, 0, 2500, 5, 1030, 0], np.int64)
    rp = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([rng.integers(0, 4000, k) for k in lens])
    out["long_rows"] = (rp, cols, len(lens), 4000)
    # repeated (r, c)
    lens = rng.integers(1, 8, 500)
    rp = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([np.full(k, rng.integers(0, 50)) if i % 3 == 0 else rng.integers(0, 50, k)
                           for i, k in enumerate(lens)])
    out["repeated"] = (rp, cols, 500, 50)
    # tiles that span thousands of empty rows: blocks of 5000 empty rows between dense rows
    lens = np.zeros(40000, np.int64)
    lens[::5000] = 3000
    lens[-1] = 3
    rp = np.concatenate([[0], np.cumsum(lens)])
    cols = rng.integers(0, 900, int(lens.sum()))
    out["empty_runs"] = (rp, cols, len(lens), 900)
    # m != n and the empty cases
    out["wide"] = (np.array([0, 2, 2, 5]), np.array([9, 1, 0, 4, 7]), 3, 10)
    out["m0"] = (np.array([0]), np.zeros(0, np.int64), 0, 4)
    out["n0"] = (np.zeros(6, np.int64), np.zeros(0, np.int64), 5, 0)
    out["nnz0"] = (np.zeros(4, np.int64), np.zeros(0, np.int64), 3, 3)
    return out


PATTERNS = _patterns()


def _row_of(ptr, lo, hi, s):
    """csr_row_of: the largest r in [lo, hi] with ptr[r] <= s, given ptr[lo] <= s (same bisection as the kernel)"""
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if ptr[mid] <= s:
            lo = mid
        else:
            hi = mid - 1
    return lo


def kernel_rows(rowptr0, nnz, m):
    """The row diff_scatter_csr assigns to every entry, and how many tiles took the staged and the global search."""
    rows = np.full(nnz, -1, np.int64)
    staged_tiles = global_tiles = 0
    for s0 in range(0, nnz, TILE):
        last = s0 + TILE - 1 if s0 + TILE < nnz else nnz - 1
        rlo, rhi = _row_of(rowptr0, 0, m - 1, s0), _row_of(rowptr0, 0, m - 1, last)
        staged = rhi - rlo < STAGE
        staged_tiles += staged
        global_tiles += not staged
        s_ptr = rowptr0[rlo: rhi + 1] if staged else None
        for s in range(s0, last + 1):
            rows[s] = rlo + _row_of(s_ptr, 0, rhi - rlo, s) if staged else _row_of(rowptr0, rlo, rhi, s)
    return rows, staged_tiles, global_tiles


@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_kernel_row_search_matches_scipy(name):
    rp, cols, m, n = PATTERNS[name]
    A = _csr(rp, cols, m, n)
    want = A.tocoo().row                     # storage order, duplicates and column order kept
    got, staged, glob = kernel_rows(np.asarray(rp, np.int64), len(cols), m)
    assert np.array_equal(got, want)
    if name == "empty_runs":
        assert glob > 0 and staged > 0          # both searches are exercised
    if name == "long_rows":
        assert staged == -(-len(cols) // TILE)  # a row across many tiles: every tile stays staged


@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_mirror_findstructralnz_and_to_dense(api, name):
    rp, cols, m, n = PATTERNS[name]
    A = _csr(rp, cols, m, n)
    M = api.SparseMatrixCSR.from_scipy(A, device="host")
    assert M.shape == (m, n) and M.nnz == len(cols)
    rows, cc = M.findstructralnz()
    coo = A.tocoo()
    assert np.array_equal(rows, coo.row + 1) and np.array_equal(cc, coo.col + 1)
    M.nzval = np.arange(1, M.nnz + 1, dtype=np.float64)
    if len(set(zip(rows.tolist(), cc.tolist()))) == M.nnz:   # scipy sums a repeated (r, c); the mirror keeps each slot
        B = sp.csr_matrix((M.nzval, A.indices, A.indptr), shape=(m, n))
        assert np.array_equal(M.to_dense(), B.toarray())
    S = M.similar()
    assert S.rowptr is M.rowptr and S.colval is M.colval and S.nzval is not M.nzval


def _csr_mirror(api, name="random_unsorted"):
    rp, cols, m, n = PATTERNS[name]
    M = api.SparseMatrixCSR.from_scipy(_csr(rp, cols, m, n), device="cpu")
    return M


def test_route_csr_j_to_the_csr_creator(api):
    M = _csr_mirror(api)
    kind, args, _ = api._plan_route(M, M, None)
    assert kind == "csr" and args[:2] == (M.m, M.n)
    assert args[2] == M.rowptr.data_ptr() and args[3] == M.colval.data_ptr() and args[4] is None
    # the same pattern in other arrays (e.g. a copy of the prototype) and the similar() of the sparsity
    other = api.SparseMatrixCSR(M.m, M.n, M.rowptr.clone(), M.colval.clone(), M.nzval.clone())
    assert api._plan_route(other, M, None)[0] == "csr"
    assert api._plan_route(M.similar(), M, np.arange(1, M.n + 1))[0] == "csr"


def test_route_dense_j_with_csr_sparsity_to_coo(api):
    M = _csr_mirror(api)
    J = torch.zeros((M.n, M.m), dtype=torch.float64).t()
    kind, args, keep = api._plan_route(J, M, None)
    assert kind == "coo"
    m, n, nnz, rows_p, cols_p, jkind, slots, ld, cv = args
    assert (m, n, nnz, jkind, slots, ld) == (M.m, M.n, M.nnz, api.L.FDB_J_DENSE, None, M.m)
    rows, cols = M.findstructralnz()
    assert np.array_equal(keep[1], rows) and np.array_equal(keep[2], cols)


def test_route_refusals(api):
    M = _csr_mirror(api)
    other = _csr_mirror(api, "wide")
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(M, other, None)             # another CSR pattern
    rp, cols, m, n = PATTERNS["random_unsorted"]
    diff = M.colval.clone()
    diff[0] = (diff[0] % n) + 1
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(api.SparseMatrixCSR(M.m, M.n, M.rowptr, diff, M.nzval), M, None)
    csc = api.SparseMatrixCSC.from_scipy(_csr(rp, cols, m, n), device="cpu")
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(M, csc, None)               # a CSC sparsity
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(M, api.BandedMatrix(M.m, M.n, 1, 1, device="cpu"), None)
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(M, None, None)
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(csc, M, None)               # a CSC J with a CSR sparsity


def test_cacheless_form_takes_j_as_sparsity(api):
    M = _csr_mirror(api)
    assert api._has_sparsestruct(M)
    assert api._shape_of(M) == (M.m, M.n)
    assert api._j_values(M) is M.nzval
    assert api._sp_key(M) == api._j_key(M) and api._j_key(M)[0] == "csr"


def test_group_routes_csr(api, pkg, monkeypatch):
    from finitediff_jl_b200 import distributed
    M = _csr_mirror(api)
    seen = {}

    def fake_create(self, creator, opts, *args):
        seen["creator"], seen["args"] = creator, args
    monkeypatch.setattr(distributed._Group, "_create", fake_create)
    distributed.GroupJacobian(M, None, "forward", [0, 0])
    assert seen["creator"] == "csr" and seen["args"][:2] == (M.m, M.n)
