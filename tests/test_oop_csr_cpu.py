"""Host side of the out-of-place CSR Jacobian (fdb_oop_plan_create_csr / fdb_group_create_oop_csr, no GPU): the CSR form
of the zero-dropping compaction (kernels_oop.cuh: oop_tile_first_col over the row pointer, CsrForm's row search and the
pointer pass of compact_tiles) restated tile by tile and checked against scipy; the routing of the two built pairings
through finite_difference_jacobian and GroupJacobianOOP; the refusals of every other pairing; and the Julia binding's
new symbols."""
import contextlib
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sps
import torch

KTILE = 1024


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


# ---- the compaction, as the kernel computes it (0-based) ----
def _row_of(ptr, lo, hi, s):
    """csr_row_of: the largest r in [lo, hi] with ptr[r] <= s, given ptr[lo] <= s"""
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if ptr[mid] <= s:
            lo = mid
        else:
            hi = mid - 1
    return lo


def tile_first_row(rowptr0, m, t0):
    """oop_tile_first_col over the row pointer: the first row whose start is at or after t0 (row m "starts" at E)"""
    lo, hi = 0, m
    while lo < hi:
        mid = (lo + hi) >> 1
        if rowptr0[mid] < t0:
            lo = mid + 1
        else:
            hi = mid
    return lo


def kernel_compact(rowptr0, cols0, vals, m):
    """compact_tiles<kFormCsr>: (rowptr, colval, nzval) 1-based as the kernel writes them, the rows each candidate's
    quotient is read at, and how many tiles took the staged and the global row search."""
    E = len(cols0)
    out_ptr = np.full(m + 1, -1, np.int64)
    out_col, out_val, rows = [], [], np.full(E, -1, np.int64)
    staged_tiles = global_tiles = 0
    if E == 0:
        out_ptr[:] = 1
        return out_ptr, np.array(out_col, np.int64), np.array(out_val), rows, 0, 0
    base = 0
    ntiles = -(-E // KTILE)
    for tile in range(ntiles):
        t0 = tile * KTILE
        last = min(t0 + KTILE, E) - 1
        rlo, rhi = _row_of(rowptr0, 0, m - 1, t0), _row_of(rowptr0, 0, m - 1, last)
        staged = rhi - rlo < KTILE
        staged_tiles += staged
        global_tiles += not staged
        kept_before = []                    # kept entries before each position of the tile
        k = 0
        for e in range(t0, last + 1):
            rows[e] = rlo + _row_of(rowptr0[rlo:rhi + 1], 0, rhi - rlo, e) if staged else \
                _row_of(rowptr0, rlo, rhi, e)
            kept_before.append(k)
            if vals[e] != 0.0:              # NaN != 0.0: kept
                out_col.append(cols0[e] + 1)
                out_val.append(vals[e])
                k += 1
        total = k
        t1 = E + 1 if tile == ntiles - 1 else t0 + KTILE
        r = tile_first_row(rowptr0, m, t0)
        while r <= m:
            p = rowptr0[r] if r < m else E
            if p >= t1:
                break
            q = p - t0
            before = total if q >= KTILE or p >= E else kept_before[q]
            out_ptr[r] = base + before + 1
            r += 1
        base += total
    return out_ptr, np.array(out_col, np.int64), np.array(out_val), rows, staged_tiles, global_tiles


def _patterns():
    rng = np.random.default_rng(11)
    out = {}
    m, n = 2500, 1900
    lens = rng.integers(0, 7, m)
    lens[rng.random(m) < 0.25] = 0
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["sorted"] = (rp, np.concatenate([np.sort(rng.permutation(n)[:k]) for k in lens]), m, n)
    out["unsorted"] = (rp, np.concatenate([rng.permutation(n)[:k] for k in lens]), m, n)
    lens = rng.integers(1, 6, 400)
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["repeated"] = (rp, np.concatenate([np.full(k, i % 40) if i % 4 == 0 else rng.integers(0, 40, k)
                                           for i, k in enumerate(lens)]), 400, 40)
    lens = np.zeros(7000, np.int64)
    lens[[0, 3000, 6999]] = [700, 900, 2000]   # tiles across more than 1024 empty rows, and one within a row
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["empty_runs"] = (rp, rng.integers(0, 300, int(lens.sum())), 7000, 300)
    lens = np.array([3, 0, 2600, 1, 0], np.int64)   # one row longer than two tiles
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["long_row"] = (rp, rng.integers(0, 3000, int(lens.sum())), 5, 3000)
    for E in (1021, 1024, 1029, 2047, 2048, 2049):
        out[f"edge{E}"] = (np.arange(E + 1), rng.integers(0, 50, E), E, 50)
    out["wide"] = (np.array([0, 2, 2, 5]), np.array([9, 1, 0, 4, 7]), 3, 10)
    out["m0"] = (np.array([0]), np.zeros(0, np.int64), 0, 4)
    out["nnz0"] = (np.zeros(4, np.int64), np.zeros(0, np.int64), 3, 3)
    return out


PATTERNS = _patterns()


def _values(E, rng):
    """candidate values with +0.0, -0.0, NaN and +-Inf among them"""
    v = rng.standard_normal(E)
    pick = rng.random(E)
    v[pick < 0.15] = 0.0
    v[(pick >= 0.15) & (pick < 0.25)] = -0.0
    v[(pick >= 0.25) & (pick < 0.28)] = np.nan
    v[(pick >= 0.28) & (pick < 0.30)] = np.inf
    v[(pick >= 0.30) & (pick < 0.32)] = -np.inf
    return v


@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_kernel_compaction_matches_scipy(name):
    rp, cols, m, n = PATTERNS[name]
    rp, cols = np.asarray(rp, np.int64), np.asarray(cols, np.int64)
    vals = _values(len(cols), np.random.default_rng(len(cols)))
    ptr, col, val, rows, staged, glob = kernel_compact(rp, cols, vals, m)
    # the rows the quotients are read at: scipy's row of every stored entry, in storage order
    A = sps.csr_matrix((np.ones(len(cols)), cols.astype(np.int32), rp.astype(np.int32)), shape=(m, n))
    assert np.array_equal(rows, A.tocoo().row)
    # the kept entries: value not +-0.0 (NaN kept), in storage order; the row pointer counts them per row
    keep = vals != 0.0
    assert np.array_equal(col, cols[keep] + 1)
    assert np.array_equal(val.view(np.int64), vals[keep].view(np.int64))
    want_ptr = 1 + np.concatenate([[0], np.cumsum([keep[rp[r]:rp[r + 1]].sum() for r in range(m)])]).astype(np.int64)
    assert np.array_equal(ptr, want_ptr)
    if name == "empty_runs":
        assert glob > 0 and staged > 0
    if name.startswith("edge") and len(cols) > KTILE:
        assert -(-len(cols) // KTILE) >= 2


def test_sorted_rows_give_the_csc_result_converted():
    """rows of sorted, distinct columns: the CSR compaction is the CSC compaction's result converted to CSR"""
    rp, cols, m, n = PATTERNS["sorted"]
    rng = np.random.default_rng(3)
    A = sps.csr_matrix((np.ones(len(cols)), cols, rp), shape=(m, n))
    # one value per (r, c): the quotient depends on the row and the column alone
    V = sps.csr_matrix((_values(len(cols), rng), cols, rp), shape=(m, n))
    ptr, col, val, _, _, _ = kernel_compact(np.asarray(rp, np.int64), np.asarray(cols, np.int64), V.data, m)
    Vc = V.tocsc()
    keep = Vc.data != 0.0                                     # the CSC route drops its zeros in CSC order
    colptr = np.concatenate([[0], np.cumsum([keep[Vc.indptr[c]:Vc.indptr[c + 1]].sum() for c in range(n)])])
    R = sps.csc_matrix((Vc.data[keep], Vc.indices[keep], colptr), shape=(m, n)).tocsr()
    assert A.has_sorted_indices and R.has_sorted_indices
    assert np.array_equal(ptr, R.indptr + 1) and np.array_equal(col, R.indices + 1)
    assert np.array_equal(val.view(np.int64), R.data.view(np.int64))


# ---- routing ----
class FakeLib:
    """Records every fdb_*create* call as (symbol, arguments after the handle and a group's device list, without the
    opts)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            if "create" in name:
                group = name.startswith("fdb_group_create_")
                self.calls.append((name, tuple(args[3:-1] if group else args[1:-1])))
            return 0
        return fn


@pytest.fixture
def fake(pkg, monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(pkg._lib, "lib", lambda: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


def _csr(api, name="unsorted"):
    rp, cols, m, n = PATTERNS[name]
    A = sps.csr_matrix((np.ones(len(cols)), cols, rp), shape=(m, n))
    return api.SparseMatrixCSR.from_scipy(A, device="cpu")


def _csc(api, name="sorted"):
    rp, cols, m, n = PATTERNS[name]
    return api.SparseMatrixCSC.from_scipy(sps.csr_matrix((np.ones(len(cols)), cols, rp), shape=(m, n)).tocsc(),
                                          device="cpu")


def _routes(api, fdist, fake, sp, proto, colorvec, fdtype="forward"):
    """(single-plan call, group call) of finite_difference_jacobian's plan and GroupJacobianOOP's members"""
    kind, pm, pn = api._oop_kind(sp, proto)
    assert kind == api.L.FDB_OOP_SPARSE and (pm, pn) == sp.shape
    csr = api._oop_csr(sp, proto)
    assert csr
    n = sp.shape[1]
    cache = object.__new__(api.JacobianCache)
    cache.fdtype, cache._plans, cache._plan_kw = fdtype, {}, {}
    fake.calls.clear()
    cvv = range(1, n + 1) if colorvec is None else colorvec
    plan = cache._oop_plan_for(kind, sp, cvv, pn, pm, n, torch.device("cuda", 0), csr)
    assert cache._oop_plan_for(kind, sp, cvv, pn, pm, n, torch.device("cuda", 0), csr) is plan   # cached
    (single,) = fake.calls
    fake.calls.clear()
    fdist.GroupJacobianOOP([0, 0], fdtype, colorvec=colorvec, sparsity=sp, jac_prototype=proto)._build(pm, n)
    (group,) = fake.calls
    return single, group


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_csr_sparsity_routes_to_the_csr_creators(api, fdist, fake, fdtype):
    M = _csr(api)
    proto = M.similar()
    cv = np.arange(M.n, dtype=np.int64) % 5 + 1
    for colorvec in (cv, None):
        single, group = _routes(api, fdist, fake, M, proto, colorvec, fdtype)
        assert single[0] == "fdb_oop_plan_create_csr" and group[0] == "fdb_group_create_oop_csr"
        assert single[1] == group[1]
        m, n, rp, cvp, colp, kind, ld = single[1]
        assert (m, n, kind, ld) == (M.m, M.n, api.L.FDB_OOP_SPARSE, M.m)
        assert rp == M.rowptr.data_ptr() and cvp == M.colval.data_ptr()     # the sparsity's own arrays
        assert (colp is None) == (colorvec is None)                         # colorvec None (1:n) is NULL


def test_csc_sparsity_arrives_transposed(api, fdist, fake):
    S = _csc(api)
    rp, cols, m, n = PATTERNS["sorted"]
    proto = _csr(api, "unsorted")                       # only the prototype's type and size matter
    seen = {}
    real = api._index_ptr

    def spy(a):
        p, keep = real(a)
        if p is not None:
            seen[p] = np.array(keep if isinstance(keep, np.ndarray) else keep.numpy())
        return p, keep
    try:
        api._index_ptr = spy
        single, group = _routes(api, fdist, fake, S, proto, None)
    finally:
        api._index_ptr = real
    assert single[0] == "fdb_oop_plan_create_csr" and group[0] == "fdb_group_create_oop_csr"
    assert single[1][:2] == (m, n) and group[1][:2] == (m, n)
    rowptr, colval = seen[single[1][2]], seen[single[1][3]]
    T = sps.csc_matrix((np.ones(len(cols)), np.asarray(S.rowval) - 1, np.asarray(S.colptr) - 1), shape=(m, n)).tocsr()
    assert np.array_equal(rowptr, T.indptr + 1) and np.array_equal(colval, T.indices + 1)
    assert np.array_equal(rowptr, np.asarray(rp) + 1) and np.array_equal(colval, np.asarray(cols) + 1)


def test_csc_prototype_and_csr_prototype_take_different_plans(api, fake):
    S = _csc(api)
    n = S.shape[1]
    cache = object.__new__(api.JacobianCache)
    cache.fdtype, cache._plans, cache._plan_kw = "forward", {}, {}
    for proto in (_csr(api, "sorted"), S):
        kind, pm, pn = api._oop_kind(S, proto)
        cache._oop_plan_for(kind, S, range(1, n + 1), pn, pm, n, torch.device("cuda", 0), api._oop_csr(S, proto))
    assert [c[0] for c in fake.calls] == ["fdb_oop_plan_create_csr", "fdb_oop_plan_create_csc"]


def test_rows_come_from_the_sparsity(api):
    M = _csr(api, "wide")
    _, rows = api._oop_rows(None, None, api.L.FDB_CENTRAL, None, 99, M, None, M.n)
    assert rows == M.m
    with pytest.raises(ValueError):
        api._oop_kind(M, _csr(api, "m0").similar())
    big = api.SparseMatrixCSR(M.m + 1, M.n, torch.ones(M.m + 2, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                              torch.zeros(0, dtype=torch.float64))
    with pytest.raises(ValueError):
        api._oop_kind(M, big)
    with pytest.raises(ValueError):
        api._oop_kind(_csc(api, "wide"), big)


def test_every_other_csr_pairing_raises(api, fdist, fake, monkeypatch):
    M = _csr(api)
    S = _csc(api, "unsorted")
    n = M.n
    dense = torch.zeros((M.n, M.m), dtype=torch.float64).t()
    band = api.BandedMatrix(M.m, M.n, 1, 1, device="cpu")
    rb = [2, 3, 4]
    block = api.BlockSkylineMatrix(rb, rb, (1, 1), device="cpu")
    bproto = api.SparseMatrixCSR(9, 9, torch.ones(10, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                                 torch.zeros(0, dtype=torch.float64))
    bandproto = api.SparseMatrixCSR(M.m, M.n, torch.ones(M.m + 1, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                                    torch.zeros(0, dtype=torch.float64))
    refused = [(M, None), (M, dense), (M, S), (None, M), (band, bandproto), (block, bproto)]
    for sp, proto in refused:
        with pytest.raises(TypeError, match="not built"):
            api._oop_kind(sp, proto)
        with pytest.raises(TypeError, match="not built"):
            fdist.GroupJacobianOOP([0, 0], "forward", sparsity=sp, jac_prototype=proto)
    # through the public entry point: refused before any device work or f call
    calls = []
    x = torch.zeros(n, dtype=torch.float64)
    monkeypatch.setattr(api, "_is_cuda", lambda t: True)
    cache = object.__new__(api.JacobianCache)
    cache.fdtype, cache._plans, cache._plan_kw = "central", {}, {}
    cache.colorvec, cache.sparsity, cache.x1, cache.fx = range(1, n + 1), None, x.clone(), torch.zeros(M.m)
    for sp, proto in refused:
        with pytest.raises(TypeError, match="not built"):
            api.finite_difference_jacobian(lambda v: calls.append(1), x, cache, sparsity=sp, jac_prototype=proto)
    assert calls == [] and fake.calls == []


def test_the_in_place_routes_do_not_change(api):
    M = _csr(api)
    S = api.SparseMatrixCSC.from_scipy(sps.csr_matrix((np.ones(M.nnz), np.asarray(M.colval) - 1,
                                                       np.asarray(M.rowptr) - 1), shape=M.shape), device="cpu")
    with pytest.raises(TypeError, match="not built"):
        api._plan_route(M, S, None)                     # a CSR J with a CSC sparsity stays refused
    assert api._plan_route(M, M, None)[0] == "csr"


def test_julia_binding_binds_the_new_entries():
    src = (Path(__file__).resolve().parent.parent / "finitediff.jl_b200" / "julia" / "FiniteDiffB200.jl").read_text()
    for sym in ("fdb_oop_plan_create_csr", "fdb_group_create_oop_csr"):
        assert f"(:{sym}, libfdjac)" in src, sym
    for needle in ("function group_oop_csr(", "function oopcsr(", "DeviceCSR(m, n, colptr, rowval[1:k], nzval[1:k])"):
        assert needle in src, needle
    hdr = (Path(__file__).resolve().parent.parent / "include" / "fdjac_b200.h").read_text()
    assert "fdb_status fdb_oop_plan_create_csr(" in hdr and "fdb_status fdb_group_create_oop_csr(" in hdr


def _julia_function(src, name):
    """the text of `function name(...) ... end` (top level: ends at the first line that is exactly `end`)"""
    i = src.index(f"\nfunction {name}(")
    j = src.index("\nend\n", i)
    return src[i:j + 5]


def test_julia_csr_plans_are_cached_on_the_pattern():
    """the CSR of a CSC sparsity is built inside the plan cache's closure, and the plan is anchored and keyed on the
    pattern's own arrays, so a repeated call reuses its plan instead of transposing, uploading and building again"""
    src = (Path(__file__).resolve().parent.parent / "finitediff.jl_b200" / "julia" / "FiniteDiffB200.jl").read_text()
    plan = _julia_function(src, "oop_csr_plan")
    closure = plan[plan.index("cached_plan(anchor, (:oop_csr"):]
    assert "csrarrays(src)" in closure and "csrarrays" not in plan[:plan.index("cached_plan(")]
    assert "anchor, second = csrid(src)" in plan and "objectid(second)" in plan
    assert "csrid(A::SparseMatrixCSC) = (A.colptr, A.rowval)" in src
    assert "transpose" in _julia_function(src, "csrarrays")
    jac = _julia_function(src, "finite_difference_jacobian")
    assert "oop_csr_plan(csr, m, n, colorvec, fd)" in jac
    for name in ("oopcsr", "finite_difference_jacobian"):
        body = _julia_function(src, name)
        assert "transpose" not in body and "csrarrays" not in body and "CuVector{Int64}(T." not in body, name
    # no sparsity, or another size: refused with the documented errors, before any size() of nothing
    oop = _julia_function(src, "oopcsr")
    assert oop.index("ArgumentError") < oop.index("size(jac_prototype)") and "DimensionMismatch" in oop
