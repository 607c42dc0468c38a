"""Host side of the banded out-of-place Jacobian (fdb_oop_plan_create_banded, no GPU): the closed forms its kernels use
(kernels_oop.cuh: band_col_start, band_locate, band_first_col, count_band_conflicts), restated here and checked against
the enumerated entry set E(m, n, l, u) and a brute-force conflict count; and the routing of every band sparsity and
prototype through finite_difference_jacobian and GroupJacobianOOP, with the TypeErrors that stay."""
import contextlib
import ctypes as C

import numpy as np
import pytest
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


# ---- the closed forms, as the kernels compute them (0-based) ----
def clamp_bands(m, n, l, u):
    return min(l, max(m - 1, 0)), min(u, n - 1)


def col_start(m, l, u, c):
    if m <= 0:
        return 0
    k = min(c, m + u)
    K = m - 1
    t = min(max(K - l + 1, 0), k)
    A = t * l + t * (t - 1) // 2 + (k - t) * K
    s = max(k - u - 1, 0)
    return k + A - s * (s + 1) // 2


def shape(m, n, l, u):
    ca = min(u, n)
    cb = max(min(m - l, n), ca)
    return dict(m=m, n=n, l=l, u=u, w=l + u + 1, ca=ca, cb=cb, sa=col_start(m, l, u, ca), sb=col_start(m, l, u, cb),
                E=col_start(m, l, u, n))


def start(b, c):
    if b["ca"] <= c <= b["cb"]:
        return b["sa"] + (c - b["ca"]) * b["w"]
    return col_start(b["m"], b["l"], b["u"], c)


def locate(b, e):
    if b["sa"] <= e < b["sb"]:
        q = e - b["sa"]
        d = q // b["w"]
        c = b["ca"] + d
        return c, c - b["u"] + (q - d * b["w"])
    lo, hi = 0, b["n"] - 1
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if col_start(b["m"], b["l"], b["u"], mid) <= e:
            lo = mid
        else:
            hi = mid - 1
    return lo, max(lo - b["u"], 0) + (e - col_start(b["m"], b["l"], b["u"], lo))


def first_col(b, t0):
    c, _ = locate(b, t0)
    return c + 1 if start(b, c) < t0 else c


def conflicts_closed_form(m, n, l, u, col):
    """count_band_conflicts: col[c] 0-based colour, < 0 for none"""
    bad = 0
    for c1 in range(n):
        if col[c1] < 0:
            continue
        hi1 = min(c1 + l, m - 1)
        for c2 in range(c1 + 1, min(c1 + l + u, n - 1) + 1):
            lo2 = max(c2 - u, 0)
            if lo2 > hi1:
                break
            if col[c2] == col[c1]:
                bad += hi1 - lo2 + 1
    return bad


# ---- the enumerated references ----
def entries(m, n, l, u):
    """E in storage order (column-major, row-sorted), unclamped bandwidths"""
    return [(r, c) for c in range(n) for r in range(max(0, c - u), min(m - 1, c + l) + 1)]


def conflicts_brute(m, n, l, u, col):
    """count_color_conflicts on the CSC of E: pairs of entries of one row whose columns share a valid colour"""
    rows = [[] for _ in range(m)]
    for r, c in entries(m, n, l, u):
        rows[r].append(c)
    bad = 0
    for cs in rows:
        for i, a in enumerate(cs):
            if col[a] < 0:
                continue
            bad += sum(1 for b in cs[i + 1:] if col[b] == col[a])
    return bad


def _cases():
    rng = np.random.default_rng(11)
    cases = [(m, n, l, u) for m in range(0, 4) for n in range(1, 4) for l in range(0, 4) for u in range(0, 4)]
    for _ in range(60):
        m, n = (int(v) for v in rng.integers(1, 300, 2))
        l, u = (int(v) for v in rng.integers(0, 40, 2))
        if rng.random() < 0.2:
            l, u = l + m, u + n          # wider than the matrix
        cases.append((m, n, l, u))
    cases += [(5000, 5000, 1, 1), (3000, 1000, 0, 7), (1000, 3000, 9, 0), (2049, 2049, 64, 64)]
    return cases


@pytest.mark.parametrize("m,n,l,u", _cases())
def test_closed_forms_enumerate_the_band(m, n, l, u):
    E = entries(m, n, l, u)
    lc, uc = clamp_bands(m, n, l, u)
    assert entries(m, n, lc, uc) == E                      # clamping keeps the entry set
    b = shape(m, n, lc, uc)
    assert b["E"] == len(E)
    starts = np.zeros(n + 1, dtype=np.int64)
    for _, c in E:
        starts[c + 1] += 1
    starts = np.cumsum(starts)
    assert [start(b, c) for c in range(n + 1)] == starts.tolist()
    assert [col_start(m, lc, uc, c) for c in range(n + 1)] == starts.tolist()
    step = max(1, len(E) // 3000)
    for e in list(range(0, len(E), step)) + list(range(max(0, len(E) - 40), len(E))):
        r, c = E[e]
        assert locate(b, e) == (c, r), (e, E[e])
        # kCopy reads candidate e from slot u + r - c of column c in the band data
        assert 0 <= uc + r - c < b["w"]
    for t0 in range(0, len(E), KTILE):                     # the first column of each tile
        assert first_col(b, t0) == int(np.searchsorted(starts[:n], t0, side="left")), t0


@pytest.mark.parametrize("m,n,l,u", [c for c in _cases() if c[0] * c[1] <= 90000])
def test_conflict_count_matches_brute_force(m, n, l, u):
    rng = np.random.default_rng(m * 7919 + n * 31 + l * 7 + u)
    lc, uc = clamp_bands(m, n, l, u)
    colourings = [np.arange(n) % (lc + uc + 1), np.arange(n) % max(1, lc + uc), rng.integers(-1, 4, n),
                  np.zeros(n, dtype=np.int64), np.full(n, -1)]
    for col in colourings:
        assert conflicts_closed_form(m, n, lc, uc, col) == conflicts_brute(m, n, l, u, col)
    # the skipped case: a cyclic colouring with more than l + u colours has no conflict
    for C in range(lc + uc + 1, lc + uc + 4):
        assert conflicts_brute(m, n, l, u, np.arange(n) % C) == 0


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


def _csc(pkg, m, n):
    cp = torch.ones(n + 1, dtype=torch.int64)
    return pkg.SparseMatrixCSC(m, n, cp, torch.zeros(0, dtype=torch.int64), None)


def _band_types(pkg, n):
    return [
        ("banded", pkg.BandedMatrix(n, n, 2, 1, device="cpu"), n, 2, 1),
        ("banded m != n", pkg.BandedMatrix(n + 3, n, 0, 4, device="cpu"), n + 3, 0, 4),
        ("banded wider than the matrix", pkg.BandedMatrix(n, n, 3 * n, 2 * n, device="cpu"), n, 3 * n, 2 * n),
        ("diagonal", pkg.Diagonal(n, device="cpu"), n, 0, 0),
        ("bidiagonal U", pkg.Bidiagonal(n, "U", device="cpu"), n, 0, 1),
        ("bidiagonal L", pkg.Bidiagonal(n, ":L", device="cpu"), n, 1, 0),
        ("symtridiagonal", pkg.SymTridiagonal(n), n, 1, 1),
    ]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_band_sparsities_route_to_the_banded_creator(pkg, api, fdist, fake, fdtype):
    n = 6
    cv = np.array([1, 2, 3, 1, 2, 3], dtype=np.int64)
    for name, sp, m, l, u in _band_types(pkg, n):
        protos = [(None, pkg._lib.FDB_OOP_DENSE), (pkg.zeros_colmajor(m, n, "cpu"), pkg._lib.FDB_OOP_DENSE),
                  (_csc(pkg, m, n), pkg._lib.FDB_OOP_SPARSE)]
        for proto, want_kind in protos:
            for colorvec in (cv, None):
                kind, pm, pn = api._oop_kind(sp, proto)
                assert kind == want_kind and (pm, pn) == (m, n) or proto is None, name
                cache = object.__new__(api.JacobianCache)
                cache.fdtype, cache._plans, cache._plan_kw = fdtype, {}, {}
                fake.calls.clear()
                cvv = range(1, n + 1) if colorvec is None else colorvec
                plan = cache._oop_plan_for(kind, sp, cvv, pn, m, n, torch.device("cuda", 0))
                assert cache._oop_plan_for(kind, sp, cvv, pn, m, n, torch.device("cuda", 0)) is plan
                (single,) = fake.calls
                fake.calls.clear()
                fdist.GroupJacobianOOP([0, 0], fdtype, colorvec=colorvec, sparsity=sp, jac_prototype=proto)._build(m, n)
                (group,) = fake.calls
                assert single[0] == "fdb_oop_plan_create_banded", name
                assert group[0] == "fdb_group_create_oop_banded", name
                assert single[1] == group[1], name
                assert single[1][:4] == (m, n, l, u), name
                assert single[1][-2:] == (kind, max(m, 1)), name
                assert (single[1][4] is None) == (colorvec is None), name


def test_band_rows_come_from_the_sparsity(pkg, api):
    n = 5
    for name, sp, m, _, _ in _band_types(pkg, n):
        f_in, rows = api._oop_rows(None, None, pkg._lib.FDB_CENTRAL, None, 99, sp, None, n)
        assert rows == m, name
        with pytest.raises(ValueError):
            api._oop_rows(None, None, pkg._lib.FDB_CENTRAL, None, 99, sp, None, n + 1)
    with pytest.raises(ValueError):
        api._oop_kind(pkg.Diagonal(n, device="cpu"), pkg.zeros_colmajor(n + 1, n, "cpu"))


def test_the_typeerrors_that_stay(pkg, api):
    n = 5
    refused_sparsities = [
        pkg.Tridiagonal(n, device="cpu"),                                              # Julia binding only
        pkg.BandedBlockBandedMatrix([2, 3], [2, 3], (1, 1), (0, 1), device="cpu"),    # a follow-up
        pkg.BandedMatrix(n, n, -1, 2, device="cpu"),                                  # negative bandwidths
        pkg.BandedMatrix(n, n, 2, -1, device="cpu"),
    ]
    for sp in refused_sparsities:
        with pytest.raises(TypeError):
            api._oop_kind(sp, None)
    structured_protos = [pkg.BandedMatrix(n, n, 1, 1, device="cpu"), pkg.Diagonal(n, device="cpu"),
                         pkg.Tridiagonal(n, device="cpu")]
    for proto in structured_protos:
        with pytest.raises(TypeError):
            api._oop_kind(pkg.BandedMatrix(n, n, 1, 1, device="cpu"), proto)


# ---- the f and the checks of the oracle-held band tests (tests/test_gpu_oop_banded.py) ----
def _oracle_shapes():
    return [(37, 37, 2, 1), (40, 37, 3, 1), (33, 37, 0, 2), (37, 37, 40, 74), (37, 37, 0, 0), (290, 300, 4, 3)]


@pytest.mark.parametrize("n,m,l,u", [(n, m, l, u) for m, n, l, u in _oracle_shapes()])
def test_band_ell_reads_exactly_the_band(n, m, l, u):
    from test_gpu_oop_banded import band_cp_rv, band_ell, band_entries
    r, c = band_entries(m, n, l, u)
    assert list(zip(r.tolist(), c.tolist())) == entries(m, n, l, u)
    cp, rv = band_cp_rv(m, n, l, u)
    assert np.array_equal(rv - 1, r) and np.array_equal(np.repeat(np.arange(n), np.diff(cp)), c)
    ell = band_ell(m, n, l, u, 3)
    listed = {(i, int(ell.cols[p, i])) for p in range(ell.K) for i in range(m)}
    assert listed == set(zip(r.tolist(), c.tolist()))
    nz = ell.coef[ell.coef != 0]
    assert np.all(np.abs(nz) >= 0.5) and np.all(np.abs(nz) <= 2.0)
    if len(r) > 500:
        share = 1 - np.count_nonzero(ell.coef) / len(r)
        assert 0.05 < share < 0.15, share


def test_band_tile_shapes_reach_their_boundaries():
    from test_gpu_oop_banded import BAND_TILES, band_entries
    assert [s[0] for s in BAND_TILES] == [1023, 1024, 1025, 2047, 2049]
    for E, m, n, l, u in BAND_TILES:
        assert m != n and len(band_entries(m, n, l, u)[0]) == E
        lens = np.diff(band_cp_rv_of(m, n, l, u))
        assert lens[0] < lens.max() and lens[-1] < lens.max(), (E, m, n, l, u)       # clipped head and tail columns


def band_cp_rv_of(m, n, l, u):
    from test_gpu_oop_banded import band_cp_rv
    return band_cp_rv(m, n, l, u)[0]


@pytest.mark.parametrize("fd,dir", [("forward", 1.0), ("forward", -1.0), ("central", 1.0), ("central", -1.0),
                                    ("complex", 1.0)])
def test_oracle_within_the_band_check(pkg, oracle, fd, dir):
    """The restatement on the band f lands within the analytic tolerance, its exact zeros (zero coefficients) give +0.0
    in the dense result; a swapped entry, an entry moved out of the band, and a -0.0 left in place of a structural zero
    each fail check_band_dense."""
    from oop_oracle import fd_oop_oracle as OO
    from test_gpu_oop_banded import _valid_cv, band_cp_rv, band_ell, band_x, check_band_dense
    from test_gpu_oop_random import Twin
    m, n, l, u = 66, 64, 4, 2
    ell = band_ell(m, n, l, u, 5)
    x = band_x(n, 6)
    cp, rv = band_cp_rv(m, n, l, u)
    cv = _valid_cv(n, l, u, m)
    cv[::9] = 0
    C_ = int(cv.max())
    eps = None if fd == "complex" else np.full(C_, (1e-7 if fd == "forward" else 6e-6) * dir)
    kw = {} if fd == "complex" else {"dir": dir, "eps_override": list(eps)}
    want = OO.jacobian_oop(Twin(ell, oracle, fd == "complex"), x, fd, None, sparsity=(m, n, cp, rv), colorvec=cv,
                           jac_prototype=("sparse", m, n), **kw)
    J = np.zeros((m, n))
    cols = np.repeat(np.arange(n), np.diff(want[3]))
    J[want[4] - 1, cols] = 0.0 + want[5]
    assert len(want[4]) < len(rv)                            # the exact zeros were dropped
    check_band_dense(J, ell, x, cv, eps, fd, m, n, l, u, "restatement")
    # a structural zero: a zero coefficient outside the row's slot 0, in a coloured column
    z = [(i, int(ell.cols[p, i])) for p in range(1, ell.K) for i in range(m)
         if ell.coef[p, i] == 0 and cv[ell.cols[p, i]] >= 1 and ell.cols[p, i] != ell.cols[0, i]]
    assert z
    r0, c0 = z[0]
    c1 = next(c for c in range(max(0, r0 - l), min(n - 1, r0 + u) + 1) if J[r0, c] != 0 and J[r0, c] != J[r0, c0])
    out = (r0 + l + 1, c0) if r0 + l + 1 < m and r0 + l + 1 > c0 + l else (0, n - 1)
    for what, edit in (("-0.0 left", lambda A: A.__setitem__((r0, c0), -0.0)),
                       ("swapped", lambda A: A.__setitem__(([r0, r0], [c0, c1]), A[[r0, r0], [c1, c0]])),
                       ("moved out", lambda A: A.__setitem__(out, A[r0, c1]))):
        bad = J.copy()
        edit(bad)
        with pytest.raises(AssertionError):
            check_band_dense(bad, ell, x, cv, eps, fd, m, n, l, u, what)
