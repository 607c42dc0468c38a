"""The banded out-of-place Jacobian on the device (fdb_oop_plan_create_banded / fdb_group_create_oop_banded, through
finite_difference_jacobian and GroupJacobianOOP) against the CSC route given the CSC of the same entry set E: the result,
the status and the f calls must be identical.  The CSC route is itself held to oop_oracle/ bit for bit
(tests/test_gpu_oop.py, tests/test_gpu_oop_random.py), so equality with it is parity with the reference's restatement.

Every compare is a bit compare of NaN-prefilled outputs.  Covered: dense, dense-prototype and sparse results in forward,
central and complex mode; dir +-1 and 0.3; step overrides; f_in; cyclic, random and invalid colourings, colour-less
columns and maximum(colorvec) < 1; every band type, m != n, l or u = 0, bands wider than the matrix; m = 0; candidate
counts at the 1024-entry tile boundaries; FDB_SM_COUNT=1; batches small enough for the candidate-copy path; groups of
1-3 members (and two GPUs when present); the refusals before any f call; the calls check_call refuses; and a sparse result
at n = 10^7 with its plan build time.

The last section holds the band route to oop_oracle/ directly, with an f whose dependence is exactly the band, and dense
results to the analytic derivative.  Results past 2^31 entries are not taken: the sparse result alone needs 16 bytes
per entry and, with the f slabs, more than 60 GB."""
import ctypes as C
import time

import numpy as np
import pytest

from _util import assert_same_bits, fdb_env

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


def make_f(m, n):
    """y_i = x_a * x_b - 3 x_c + 0.5 x_a with a = i mod n, b = (i+1) mod n, c = (i+2) mod n: every op a single IEEE op on
    gathered components (analytic, so the complex step applies); records every point it sees"""
    idx = [torch.arange(m, device="cuda") % max(n, 1), (torch.arange(m, device="cuda") + 1) % max(n, 1),
           (torch.arange(m, device="cuda") + 2) % max(n, 1)]

    def fn(x):
        if fn.record:
            fn.points.append(x.detach().cpu().numpy().copy())
        if m == 0:
            return torch.zeros(0, dtype=x.dtype, device=x.device)
        a, b, c = (x[i] for i in idx)
        return (a * b - 3.0 * c) + 0.5 * a

    fn.points, fn.record = [], True
    return fn


def band_csc(pkg, m, n, l, u):
    cols = [np.arange(max(0, c - u), min(m - 1, c + l) + 1, dtype=np.int64) for c in range(n)]
    colptr = np.concatenate([[1], 1 + np.cumsum([len(r) for r in cols])]).astype(np.int64)
    rowval = (np.concatenate(cols) + 1).astype(np.int64) if cols else np.zeros(0, np.int64)
    return pkg.SparseMatrixCSC(m, n, torch.from_numpy(colptr), torch.from_numpy(rowval), None)


def sparse_proto(pkg, m, n):
    return pkg.SparseMatrixCSC(m, n, torch.ones(n + 1, dtype=torch.int64), torch.zeros(0, dtype=torch.int64), None)


def host(res):
    if isinstance(res, torch.Tensor):
        return ("dense", res.cpu().numpy())
    return ("sparse", res.m, res.n, res.colptr.cpu().numpy(), res.rowval.cpu().numpy(), res.nzval.cpu().numpy())


def assert_same(got, want, what):
    g, w = host(got), host(want)
    assert g[0] == w[0], what
    if g[0] == "dense":
        assert_same_bits(g[1], w[1], f"{what}: J")
        return
    assert g[1:3] == w[1:3], what
    assert np.array_equal(g[3], w[3]), f"{what}: colptr"
    assert np.array_equal(g[4], w[4]), f"{what}: rowval"
    assert_same_bits(g[5], w[5], f"{what}: nzval")


def _x(n, seed=0):
    x = np.random.default_rng(seed).uniform(-1.5, 1.5, n)
    if n > 3:
        x[1], x[2] = -0.0, 0.0
    return torch.from_numpy(x).cuda()


def run_pair(pkg, sp, m, n, l, u, kind, fd, cv, *, dir=1.0, relstep=None, absstep=None, f_in=False, seed=0, **plan_kw):
    """(band result, CSC result) and the points each f saw; x unchanged afterwards"""
    x = _x(n, seed)
    x0 = x.clone()
    out = []
    for which in ("band", "csc"):
        sparsity = sp if which == "band" else band_csc(pkg, m, n, l, u)
        proto = {"dense": None, "dense_proto": torch.full((n, m), float("nan"), dtype=torch.float64, device="cuda").t(),
                 "sparse": sparse_proto(pkg, m, n)}[kind]
        f = make_f(m, n)
        fx = torch.zeros(m, dtype=torch.float64, device="cuda")
        cache = pkg.JacobianCache(x, fx, fd, **plan_kw)
        fin = f(x) if f_in else None
        f.points.clear()
        res = pkg.finite_difference_jacobian(f, x, cache, fin, relstep=relstep, absstep=absstep, dir=dir,
                                             colorvec=cv, sparsity=sparsity, jac_prototype=proto)
        torch.cuda.synchronize()
        out.append((res, f.points, cache._last_plan))
        assert_same_bits(x.cpu().numpy(), x0.cpu().numpy(), "x modified")
    (rb, pb, planb), (rc, pc, planc) = out
    assert len(pb) == len(pc)
    for a, b in zip(pb, pc):
        assert_same_bits(a.view(np.float64), b.view(np.float64), "points f saw")   # complex points as (re, im) pairs
    assert planb.info()["n_entries"] == planc.info()["n_entries"]
    return rb, rc, planb


def _types(pkg, n):
    return [
        ("banded 2,1", pkg.BandedMatrix(n, n, 2, 1), n, 2, 1),
        ("banded m > n", pkg.BandedMatrix(n + 5, n, 3, 0), n + 5, 3, 0),
        ("banded m < n", pkg.BandedMatrix(max(n - 4, 1), n, 0, 2), max(n - 4, 1), 0, 2),
        ("banded wider than the matrix", pkg.BandedMatrix(n, n, n + 3, 2 * n), n, n + 3, 2 * n),
        ("diagonal", pkg.Diagonal(n), n, 0, 0),
        ("bidiagonal U", pkg.Bidiagonal(n, "U"), n, 0, 1),
        ("bidiagonal L", pkg.Bidiagonal(n, "L"), n, 1, 0),
        ("symtridiagonal", pkg.SymTridiagonal(n), n, 1, 1),
    ]


def _valid_cv(n, l, u, m):
    lc, uc = min(l, max(m - 1, 0)), min(u, n - 1)
    return (np.arange(n) % (lc + uc + 1) + 1).astype(np.int64)


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
@pytest.mark.parametrize("kind", ["dense", "dense_proto", "sparse"])
@pytest.mark.parametrize("n", [1, 2, 3, 37])
def test_every_type_matches_the_csc_route(pkg, fd, kind, n):
    for name, sp, m, l, u in _types(pkg, n):
        cv = _valid_cv(n, l, u, m)
        rb, rc, _ = run_pair(pkg, sp, m, n, l, u, kind, fd, cv)
        assert_same(rb, rc, f"{name} {kind} {fd} n={n}")


@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("kind", ["dense", "sparse"])
@pytest.mark.parametrize("dir,steps,f_in", [(1.0, (None, None), False), (-1.0, (None, None), True),
                                            (0.3, (1e-4, None), False), (1.0, (None, 1e-3), True),
                                            (-1.0, (1e-5, 1e-9), False)])
def test_step_options_match(pkg, fd, kind, dir, steps, f_in):
    n = 300
    sp = pkg.BandedMatrix(n, n, 4, 3)
    rb, rc, _ = run_pair(pkg, sp, n, n, 4, 3, kind, fd, _valid_cv(n, 4, 3, n), dir=dir, relstep=steps[0],
                         absstep=steps[1], f_in=f_in and fd == "forward")
    assert_same(rb, rc, f"{kind} {fd} dir={dir} steps={steps}")


def test_sparse_result_takes_any_colouring(pkg):
    n, m = 200, 230
    rng = np.random.default_rng(5)
    colourings = {
        "random": rng.integers(1, 6, n),
        "colour-less columns": np.where(rng.random(n) < 0.3, 0, rng.integers(1, 4, n)),
        "max < 1": np.zeros(n, dtype=np.int64),
        "negative": -np.ones(n, dtype=np.int64),
        "cyclic too few": np.arange(n) % 2 + 1,
        "identity": None,
    }
    for fd in ("forward", "central", "complex"):
        for name, cv in colourings.items():
            cvv = range(1, n + 1) if cv is None else cv.astype(np.int64)
            rb, rc, _ = run_pair(pkg, pkg.BandedMatrix(m, n, 5, 2), m, n, 5, 2, "sparse", fd, cvv)
            assert_same(rb, rc, f"{name} {fd}")


def test_dense_result_with_colourless_columns(pkg):
    n = 150
    cv = _valid_cv(n, 2, 2, n)
    cv[::7] = 0
    for fd in ("forward", "central"):
        rb, rc, _ = run_pair(pkg, pkg.BandedMatrix(n, n, 2, 2), n, n, 2, 2, "dense_proto", fd, cv)
        assert_same(rb, rc, fd)


def test_invalid_colouring_refused_before_any_f_call(pkg):
    n = 40
    for cv in (np.arange(n) % 2 + 1, np.ones(n)):
        errs = []
        for which in ("band", "csc"):
            sp = pkg.BandedMatrix(n, n, 1, 1) if which == "band" else band_csc(pkg, n, n, 1, 1)
            f = make_f(n, n)
            x = _x(n)
            cache = pkg.JacobianCache(x, "central")
            with pytest.raises(pkg._lib.FdbError) as ei:
                pkg.finite_difference_jacobian(f, x, cache, colorvec=cv.astype(np.int64), sparsity=sp)
            assert f.points == []
            errs.append((ei.value.status, str(ei.value)))
        assert errs[0] == errs[1]


@pytest.mark.parametrize("n", [341, 342, 343, 683, 1024, 1025])
def test_tile_boundaries_and_one_sm(pkg, n):
    # tridiagonal: 3n - 2 candidates = 1021, 1024, 1027, 2047, 3070, 3073
    for sm in (None, 1):
        with fdb_env(SM_COUNT=sm):
            for fd in ("forward", "central"):
                rb, rc, _ = run_pair(pkg, pkg.SymTridiagonal(n), n, n, 1, 1, "sparse", fd, _valid_cv(n, 1, 1, n))
                assert_same(rb, rc, f"n={n} sm={sm} {fd}")


def test_empty_rows(pkg):
    n = 9
    for kind in ("dense", "sparse"):
        rb, rc, _ = run_pair(pkg, pkg.BandedMatrix(0, n, 1, 1), 0, n, 1, 1, kind, "central", _valid_cv(n, 1, 1, 1))
        assert_same(rb, rc, kind)


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_candidate_copy_path(pkg, fd):
    """one f! output per group (max_batch 1, a small scratch budget): the band scatter writes band data and the compaction
    copies from it"""
    n = 2000
    for l, u in ((1, 1), (40, 33)):
        cv = _valid_cv(n, l, u, n)
        rb, rc, plan = run_pair(pkg, pkg.BandedMatrix(n, n, l, u), n, n, l, u, "sparse", fd, cv, max_batch=1,
                                scratch_bytes=1)
        assert plan.info()["n_groups"] > 1
        assert_same(rb, rc, f"l={l} u={u}")


def _band_group(pkg, fdist, devs, fd, sp, kind, m, n, cv, x, f_in=None, **kw):
    proto = sparse_proto(pkg, m, n) if kind == "sparse" else None
    g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=sp, jac_prototype=proto, **kw)
    fs = [make_f(m, n) for _ in devs]
    try:
        res = g.run(fs, x, f_in)
        torch.cuda.synchronize()
        return host(res), sum(len(f.points) for f in fs)
    finally:
        g.close()


@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_groups_match_one_device(pkg, fdist, fd, kind):
    n = 500
    sets = [[0], [0, 0], [0, 0, 0]]
    if torch.cuda.device_count() >= 2:
        sets.append([0, 1])
    for l, u, cv in ((1, 1, _valid_cv(n, 1, 1, n)), (6, 2, _valid_cv(n, 6, 2, n)), (0, 0, np.ones(n, np.int64))):
        sp = pkg.BandedMatrix(n, n, l, u)
        x = _x(n, 3)
        want, calls = _band_group(pkg, fdist, [0], fd, sp, kind, n, n, cv, x)
        single = pkg.finite_difference_jacobian(make_f(n, n), x, pkg.JacobianCache(x, fd), colorvec=cv, sparsity=sp,
                                                jac_prototype=sparse_proto(pkg, n, n) if kind == "sparse" else None)
        assert_same_tuple(host(single), want, "group [0] vs one device")
        for devs in sets[1:]:
            got, gcalls = _band_group(pkg, fdist, devs, fd, sp, kind, n, n, cv, x)
            assert gcalls == calls, devs
            assert_same_tuple(got, want, f"{devs} l={l} u={u}")
    # no valid colour: rank 0 writes the zeros of every column
    got, _ = _band_group(pkg, fdist, [0, 0], fd, pkg.BandedMatrix(n, n, 1, 1), kind, n, n, np.zeros(n, np.int64), x)
    want, _ = _band_group(pkg, fdist, [0], fd, pkg.BandedMatrix(n, n, 1, 1), kind, n, n, np.zeros(n, np.int64), x)
    assert_same_tuple(got, want, "no valid colour")


def assert_same_tuple(g, w, what):
    assert g[0] == w[0], what
    if g[0] == "dense":
        assert_same_bits(g[1], w[1], what)
        return
    assert g[1:3] == w[1:3], what
    assert np.array_equal(g[3], w[3]) and np.array_equal(g[4], w[4]), what
    assert_same_bits(g[5], w[5], what)


# ---- the C ABI directly ----
def _create(pkg, m, n, l, u, cv, kind, **opt):
    L = pkg._lib
    from finitediff_jl_b200 import api
    o = api._opts(L.FDB_FORWARD, 0, **opt)
    h = C.c_void_p()
    cvp = cv.ctypes.data if cv is not None else None
    st = L.lib().fdb_oop_plan_create_banded(C.byref(h), m, n, l, u, cvp, kind, max(m, 1), C.byref(o))
    return st, h


def test_negative_bandwidths_unsupported(pkg):
    L = pkg._lib
    for l, u in ((-1, 2), (2, -1)):
        for kind in (L.FDB_OOP_DENSE, L.FDB_OOP_SPARSE):
            st, h = _create(pkg, 10, 10, l, u, None, kind)
            assert st == L.FDB_ERR_UNSUPPORTED and not h.value
    st, h = _create(pkg, 10, 10, 1, 1, None, L.FDB_OOP_RAW)
    assert st == L.FDB_ERR_INVALID and not h.value
    st, h = _create(pkg, 10, 0, 1, 1, None, L.FDB_OOP_DENSE)
    assert st == L.FDB_ERR_INVALID and not h.value


def test_sparse_rank_plan_alone_is_refused_and_check_call_rows(pkg):
    L = pkg._lib
    n = 64
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    calls = []

    @L.FDB_FN
    def f(ctx, fx, x, batch, ldfx, ldx, stream):
        calls.append(1)
        return 0

    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    st, h = _create(pkg, n, n, 1, 1, cv, L.FDB_OOP_SPARSE, rank=0, world=2)
    assert st == L.FDB_OK
    out = L.OopOut()
    buf = [torch.empty(k, dtype=dt, device="cuda") for k, dt in ((n + 1, torch.int64), (3 * n, torch.int64),
                                                                 (3 * n, torch.float64), (1, torch.int64))]
    out.colptr, out.rowval, out.nzval, out.nnz = (b.data_ptr() for b in buf)
    out.cap = 3 * n
    st = L.lib().fdb_jacobian_oop(h, f, None, x.data_ptr(), C.byref(out), None, None, float("nan"), float("nan"), 1.0, None)
    assert st == L.FDB_ERR_INVALID and calls == []
    assert "fdb_group_create_oop_" in L.lib().fdb_last_error().decode()
    L.lib().fdb_plan_destroy(h)
    st, h = _create(pkg, n, n, 1, 1, cv, L.FDB_OOP_DENSE)
    J = torch.empty(n * n, dtype=torch.float64, device="cuda")
    st = L.lib().fdb_jacobian(h, f, None, x.data_ptr(), J.data_ptr(), None, None, float("nan"), float("nan"), 1.0, None)
    assert st == L.FDB_ERR_INVALID and calls == []
    assert L.lib().fdb_last_error().decode() == "this is an out-of-place plan: call fdb_jacobian_oop"
    L.lib().fdb_plan_destroy(h)
    g = C.c_void_p()
    devs = (C.c_int * 2)(0, 0)
    from finitediff_jl_b200 import api
    o = api._opts(L.FDB_FORWARD, 0)
    assert L.lib().fdb_group_create_oop_banded(C.byref(g), 2, devs, n, n, 1, 1, cv.ctypes.data, L.FDB_OOP_DENSE, n,
                                               C.byref(o)) == L.FDB_OK
    st = L.lib().fdb_group_jacobian(g, f, None, x.data_ptr(), J.data_ptr(), None, None, float("nan"), float("nan"), 1.0,
                                    None)
    assert st == L.FDB_ERR_INVALID and calls == []
    assert L.lib().fdb_last_error().decode() == "this is an out-of-place group: call fdb_group_jacobian_oop"
    L.lib().fdb_group_destroy(g)


def test_ten_million_columns(pkg):
    """N = 10^7, l = u = 1, 3 colours: the whole sparse result equals the CSC route's; the band plan builds in under 1 s"""
    n = 10_000_000
    L = pkg._lib
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    x = _x(n, 9)
    res = []
    for which in ("band", "csc"):
        sp = pkg.BandedMatrix(n, n, 1, 1) if which == "band" else band_csc(pkg, n, n, 1, 1)
        cache = pkg.JacobianCache(x, "forward")
        f = make_f(n, n)
        f.record = False
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        plan = cache._oop_plan_for(L.FDB_OOP_SPARSE, sp, cv, n, n, n, x.device)
        build = time.perf_counter() - t0
        if which == "band":
            assert build < 1.0, build
        r = pkg.finite_difference_jacobian(f, x, cache, colorvec=cv, sparsity=sp, jac_prototype=sparse_proto(pkg, n, n))
        assert cache._last_plan is plan
        torch.cuda.synchronize()
        res.append(r)
        del plan
    assert torch.equal(res[0].colptr, res[1].colptr) and torch.equal(res[0].rowval, res[1].rowval)
    assert torch.equal(res[0].nzval.view(torch.int64), res[1].nzval.view(torch.int64))



# ------------------------------------------------------------------------------------------------ held to oop_oracle
# The comparisons above hold the band route to the CSC route, with an f whose dependence is not the band.  Here f is the
# ELL rows function of test_gpu_oop_random.py built so that row r reads exactly the band columns max(0, r-l) ..
# min(n-1, r+u), in random order, with coefficients in +-[0.5, 2] of which about one in ten is exactly 0: those entries'
# quotients are exactly +-0 (-0.0 with dir = -1), dropped from a sparse result and +0.0 in a dense one.  Each case runs
# the band sparsity object on the device through run_csc and the restatement oop_oracle/ on the CSC of the band's entry
# set, bit for bit, with the same f calls; dense results are also held to the analytic derivative.
import test_gpu_oop_random as OR  # noqa: E402
from test_gpu_structured_fill import analytic_tolerance, ell_derivative  # noqa: E402


def band_entries(m, n, l, u):
    """(rows, cols), 0-based, of the band's entries in storage order (column-major, rows ascending)"""
    cols = [np.arange(max(0, c - u), min(m - 1, c + l) + 1, dtype=np.int64) for c in range(n)]
    r = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    c = np.repeat(np.arange(n, dtype=np.int64), [len(v) for v in cols])
    return r, c


def band_cp_rv(m, n, l, u):
    r, c = band_entries(m, n, l, u)
    cp = np.concatenate([[0], np.cumsum(np.bincount(c, minlength=n))]).astype(np.int64) + 1
    return cp, r + 1


def band_ell(m, n, l, u, seed, zero_share=0.1):
    """row r reads exactly the band columns of row r in random order; coefficients +-[0.5, 2], about zero_share of them
    exactly 0 (padding repeats the row's first column with coefficient 0)"""
    rng = np.random.default_rng(seed)
    # row r of a band holds the columns c with r - l <= c <= r + u
    rows = [np.arange(max(0, r - l), min(n - 1, r + u) + 1) for r in range(m)]
    assert all(len(v) for v in rows), "a row without a band column"
    K = max(len(v) for v in rows)
    cols = np.zeros((K, m), np.int64)
    coef = np.zeros((K, m))
    for r, v in enumerate(rows):
        v = rng.permutation(v)
        cols[:, r] = v[0]
        cols[:len(v), r] = v
        a = rng.uniform(0.5, 2.0, len(v)) * np.where(rng.random(len(v)) < 0.5, -1.0, 1.0)
        a[rng.random(len(v)) < zero_share] = 0.0
        coef[:len(v), r] = a
    return OR.Ell(cols, coef)


def check_band_dense(J, ell, x, cv, eps, fd, m, n, l, u, what):
    """Every element outside the band, and every band entry of a column without a valid colour, is +0.0 by bit pattern;
    every band entry of a coloured column is within the analytic tolerance of d f_r / d x_c (valid colourings only)."""
    J = np.asarray(J)
    assert J.shape == (m, n), what
    r, c = band_entries(m, n, l, u)
    inside = np.zeros((m, n), bool)
    inside[r, c] = True
    assert np.all(J[~inside].view(np.uint64) == 0), f"{what}: an element outside the band is not +0.0"
    k = cv[c] - 1
    live = k >= 0
    assert np.all(J[r[~live], c[~live]].view(np.uint64) == 0), f"{what}: a column without a colour is not +0.0"
    r, c, k = r[live], c[live], k[live]
    d, S, T = ell_derivative(ell.cols.astype(np.int64), ell.coef, r, c, x)
    tol = analytic_tolerance(fd, None if fd == "complex" else np.asarray(eps)[k], S, T, ell.K)
    v = J[r, c]
    bad = np.flatnonzero(~(np.abs(v - d) <= tol))
    assert bad.size == 0, (f"{what}: {bad.size} band entries off the derivative; first ({r[bad[0]]}, {c[bad[0]]}): "
                           f"{v[bad[0]]!r} vs {d[bad[0]]!r}")
    assert np.all(J[r, c][d == 0].view(np.uint64) == 0), f"{what}: a zero derivative is not +0.0"


def band_x(n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.5, 1.5, n) * np.where(rng.random(n) < 0.5, -1.0, 1.0)


def run_band(pkg, oracle, sp, m, n, l, u, cv, *, fd="forward", sparse=True, seed=0, analytic=True, nan=False, what="",
             **kw):
    """run_csc with the band object on the device and the CSC of its entries in the restatement; the dense result's
    analytic check (only for valid colourings, and x without NaN; nan: one NaN component, kept by the compaction)"""
    ell = kw.pop("ell", None) or band_ell(m, n, l, u, seed)
    x = band_x(n, seed + 1)
    if nan:
        x[n // 2] = np.nan
        analytic = False
    cp, rv = band_cp_rv(m, n, l, u)
    res, plan = OR.run_csc(pkg, oracle, ell, x, cp, rv, cv, fd=fd, sparse=sparse, band=sp, what=what, **kw)
    assert plan is None or plan.info()["n_entries"] == len(rv), what
    if res is not None and not sparse and analytic and kw.get("steps", (None, None)) == (None, None):
        eps = None if fd == "complex" else plan.eps()
        check_band_dense(res.cpu().numpy(), ell, x, cv, eps, fd, m, n, l, u, what)
    return res, plan, ell, x


def _oracle_types(pkg, n):
    """(name, band object, m, l, u): every row of each holds at least one band column"""
    return [
        ("banded 2,1", pkg.BandedMatrix(n, n, 2, 1), n, 2, 1),
        ("banded m > n", pkg.BandedMatrix(n + 3, n, 3, 1), n + 3, 3, 1),
        ("banded m < n", pkg.BandedMatrix(n - 4, n, 0, 2), n - 4, 0, 2),
        ("banded l = 0", pkg.BandedMatrix(n, n, 0, 3), n, 0, 3),
        ("banded u = 0", pkg.BandedMatrix(n, n, 4, 0), n, 4, 0),
        ("banded wider than the matrix", pkg.BandedMatrix(n, n, n + 3, 2 * n), n, n + 3, 2 * n),
        ("diagonal", pkg.Diagonal(n), n, 0, 0),
        ("bidiagonal U", pkg.Bidiagonal(n, "U"), n, 0, 1),
        ("bidiagonal L", pkg.Bidiagonal(n, "L"), n, 1, 0),
        ("symtridiagonal", pkg.SymTridiagonal(n), n, 1, 1),
    ]


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
def test_band_types_against_the_oracle(pkg, oracle, fd, sparse):
    for n in (5, 37, 130):
        for name, sp, m, l, u in _oracle_types(pkg, n):
            cv = _valid_cv(n, l, u, m)
            what = f"{name} n={n} {fd} sparse={sparse}"
            res, _, ell, x = run_band(pkg, oracle, sp, m, n, l, u, cv, fd=fd, sparse=sparse, seed=n, what=what)
            if not sparse:
                # the dense prototype takes the same values
                xd = torch.from_numpy(x).cuda()
                f, _ = ell.native(pkg, fd == "complex")
                proto = torch.full((n, m), float("nan"), dtype=torch.float64, device="cuda").t()
                cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd)
                got = pkg.finite_difference_jacobian(f, xd, cache, colorvec=cv, sparsity=sp, jac_prototype=proto)
                torch.cuda.synchronize()
                assert_same_bits(got.cpu().numpy(), res.cpu().numpy(), f"{what}: dense prototype")


BAND_OPTIONS = [("dir+", dict(dir=1.0)), ("dir-", dict(dir=-1.0)), ("steps", dict(steps=(1e-5, 1e-9))),
                ("abs0", dict(steps=(None, 0.0))), ("f_in", dict(f_in=True)), ("f_in dir-", dict(f_in=True, dir=-1.0)),
                ("nan", dict(nan=True))]


@pytest.mark.parametrize("opt", BAND_OPTIONS, ids=[o[0] for o in BAND_OPTIONS])
@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
def test_band_options_against_the_oracle(pkg, oracle, opt, fd, sparse):
    name, kw = opt
    if kw.get("f_in") and fd != "forward":
        pytest.skip("f_in is the forward mode's f(x)")
    n, m, l, u = 300, 290, 4, 3
    cv = _valid_cv(n, l, u, m)
    cv[::11] = 0
    res, plan, ell, x = run_band(pkg, oracle, pkg.BandedMatrix(m, n, l, u), m, n, l, u, cv, fd=fd, sparse=sparse,
                                 seed=17, what=f"{name} {fd} sparse={sparse}", **kw)
    if sparse:
        # the exact zeros (zero coefficients, columns without a colour) are dropped; NaN quotients are kept
        assert res.nnz < len(band_entries(m, n, l, u)[0]), name
        if kw.get("nan"):
            assert np.isnan(res.nzval.cpu().numpy()).any(), name


def _cyclic_many():
    n, l, u = 3000, 700, 400
    cv = _valid_cv(n, l, u, n)
    assert cv.max() == 1101
    return n, l, u, cv


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_band_many_colours(pkg, oracle, fd):
    """1101 cyclic colours (the closed form) and their relabelling (a 16-bit table), sparse against the restatement;
    the dense result equals the sparse one scattered into +0.0 and meets the analytic check"""
    n, l, u, cv = _cyclic_many()
    ell = band_ell(n, n, l, u, 81)
    sp = pkg.BandedMatrix(n, n, l, u)
    for cvname, c in (("cyclic", cv), ("relabelled", 1102 - cv))[:2 if fd == "forward" else 1]:
        what = f"C=1101 {cvname} {fd}"
        res, plan, _, x = run_band(pkg, oracle, sp, n, n, l, u, c, fd=fd, sparse=True, seed=81, ell=ell, max_batch=4,
                                   record=False, native_twin=True, what=what)
        info = plan.info()
        assert info["n_colors"] == 1101 and info["color_bits"] == 16, info
        xd = torch.from_numpy(x).cuda()
        f, _ = ell.native(pkg, fd == "complex")
        cache = pkg.JacobianCache(xd, torch.zeros(n, dtype=torch.float64, device="cuda"), fd, max_batch=4)
        J = pkg.finite_difference_jacobian(f, xd, cache, colorvec=c, sparsity=sp)
        torch.cuda.synchronize()
        h = _host_sparse(res)
        want = np.zeros((n, n))
        want[h[0], h[1]] = 0.0 + h[2]
        assert_same_bits(J.cpu().numpy(), want, f"{what}: dense vs sparse")
        check_band_dense(J.cpu().numpy(), ell, x, c, None if fd == "complex" else cache._last_plan.eps(), fd, n, n, l, u,
                         what)


def test_band_many_colours_identity(pkg, oracle):
    """the identity colouring past 1024 colours, sparse result, on a narrow band (f runs once per column)"""
    n, m, l, u = 1100, 1103, 3, 2
    _, plan, _, _ = run_band(pkg, oracle, pkg.BandedMatrix(m, n, l, u), m, n, l, u, np.arange(1, n + 1), seed=83,
                             max_batch=8, record=False, native_twin=True, what="identity n=1100")
    assert plan.info()["n_colors"] == 1100 and plan.info()["color_bits"] == 16


def _host_sparse(res):
    cp = res.colptr.cpu().numpy()
    cols = np.repeat(np.arange(len(cp) - 1), np.diff(cp))
    return res.rowval.cpu().numpy() - 1, cols, res.nzval.cpu().numpy()


@pytest.mark.parametrize("spread", [300, 70_000], ids=["16bit", "32bit"])
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
def test_band_wide_colour_tables(pkg, oracle, spread, sparse):
    """colour ids spread to 300 or 70 000 (a valid colouring stays valid, so the dense result takes them too)"""
    n, m, l, u = 60, 64, 4, 2
    rng = np.random.default_rng(spread)
    cv = _valid_cv(n, l, u, m)
    cv[rng.random(n) < 0.1] = 0
    cv = OR.spread_ids(cv, spread, rng)
    assert cv.max() == spread
    for fd in ("forward", "central"):
        _, plan, _, _ = run_band(pkg, oracle, pkg.BandedMatrix(m, n, l, u), m, n, l, u, cv, fd=fd, sparse=sparse,
                                 seed=spread, max_batch=8, record=False, native_twin=True,
                                 dir=-1.0 if fd == "forward" else 1.0, what=f"spread {spread} {fd} sparse={sparse}")
        assert plan.info()["color_bits"] == (16 if spread == 300 else 32)


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_band_candidate_copy_against_the_oracle(pkg, oracle, fd):
    n = 2000
    for l, u in ((1, 1), (40, 33)):
        cv = _valid_cv(n, l, u, n)
        _, plan, _, _ = run_band(pkg, oracle, pkg.BandedMatrix(n, n, l, u), n, n, l, u, cv, fd=fd, seed=l,
                                 max_batch=1, scratch=1, record=False, native_twin=True, what=f"copy l={l} u={u} {fd}")
        assert plan.info()["n_groups"] > 1


def band_tile_shapes():
    """(E, m, n, l, u): band shapes with m != n, both bandwidths clipped at the matrix edges (head and tail columns of
    varying length), and E candidates at and around the 1024-entry tile boundaries"""
    def count(m, n, l, u):
        c = np.arange(n)
        return int(np.maximum(np.minimum(m - 1, c + l) - np.maximum(0, c - u) + 1, 0).sum())

    out = []
    for E in (1023, 1024, 1025, 2047, 2049):
        found = next(((E, m, n, l, u) for n in range(60, 400) for d in (5, -3, 2, -1) for l in range(5, 16)
                      for u in range(3, 16) for m in (n + d,) if count(m, n, l, u) == E), None)
        assert found, E
        out.append(found)
    return out


BAND_TILES = band_tile_shapes()


@pytest.mark.parametrize("shape", BAND_TILES, ids=[f"E{s[0]}" for s in BAND_TILES])
@pytest.mark.parametrize("sm", [None, 1])
def test_band_tiles_against_the_oracle(pkg, oracle, shape, sm):
    E, m, n, l, u = shape
    cv = _valid_cv(n, l, u, m)
    for fd in ("forward", "central"):
        for sparse in (True, False):
            _, plan, _, _ = run_band(pkg, oracle, pkg.BandedMatrix(m, n, l, u), m, n, l, u, cv, fd=fd, sparse=sparse,
                                     seed=E, sm=sm, dir=-1.0, what=f"E={E} sm={sm} {fd} sparse={sparse}")
            assert plan.info()["n_entries"] == E


def _group_sets():
    sets = [[0, 0], [0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets.append([0, 1])
    return sets


@pytest.mark.parametrize("devs", _group_sets(), ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
def test_band_groups_against_the_oracle(pkg, oracle, fdist, devs, sparse):
    """GroupJacobianOOP with colour-less columns: the group result is the one-device result, which is the restatement's"""
    n, m, l, u = 400, 405, 6, 3
    cv = _valid_cv(n, l, u, m)
    cv[::7] = 0
    sp = pkg.BandedMatrix(m, n, l, u)
    for fd in ("forward", "central"):
        for partition in (0, 1):
            what = f"group {devs} {fd} sparse={sparse} partition={partition}"
            single, plan, ell, x = run_band(pkg, oracle, sp, m, n, l, u, cv, fd=fd, sparse=sparse, seed=91,
                                            record=False, what=what)
            xd = torch.from_numpy(x).cuda(devs[0])
            proto = sparse_proto(pkg, m, n) if sparse else None
            with torch.cuda.device(devs[0]):
                g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=sp, jac_prototype=proto, partition=partition)
                members = [ell.native(pkg, device=f"cuda:{d}") for d in devs]
                try:
                    res = g.run([f for f, _ in members], xd)
                    torch.cuda.synchronize()
                finally:
                    g.close()
            assert_same_tuple(host(res), host(single), f"{what}: against one device")
            Cn = int(cv.max())
            assert sum(ctx.calls for _, ctx in members) == (2 * Cn if fd == "central" else Cn + 1), what
