"""The banded out-of-place Jacobian on the device (fdb_oop_plan_create_banded / fdb_group_create_oop_banded, through
finite_difference_jacobian and GroupJacobianOOP) against the CSC route given the CSC of the same entry set E: the result,
the status and the f calls must be identical.  The CSC route is itself held to oop_oracle/ bit for bit
(tests/test_gpu_oop.py, tests/test_gpu_oop_random.py), so equality with it is parity with the reference's restatement.

Every compare is a bit compare of NaN-prefilled outputs.  Covered: dense, dense-prototype and sparse results in forward,
central and complex mode; dir +-1 and 0.3; step overrides; f_in; cyclic, random and invalid colourings, colour-less
columns and maximum(colorvec) < 1; every band type, m != n, l or u = 0, bands wider than the matrix; m = 0; candidate
counts at the 1024-entry tile boundaries; FDB_SM_COUNT=1; batches small enough for the candidate-copy path; groups of
1-3 members (and two GPUs when present); the refusals before any f call; the calls check_call refuses; and a sparse result
at n = 10^7 with its plan build time."""
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

