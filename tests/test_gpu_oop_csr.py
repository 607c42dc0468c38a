"""The out-of-place CSR Jacobian on the device (fdb_oop_plan_create_csr / fdb_group_create_oop_csr, through
finite_difference_jacobian and GroupJacobianOOP with a SparseMatrixCSR prototype).  Every case runs the CSC route on the
CSC of the same entry set, held bit for bit to the restatement oop_oracle/ (test_gpu_oop_random.run_csc), and holds the
CSR result to it: the CSR result must be the CSC result's kept (row, column) values laid out in the CSR sparsity's own
slot order (unsorted columns and repeated pairs included), with rowptr, colval and the kept count exact and the values
compared as bit patterns.  The f calls and the points passed to f must be those of the CSC route."""
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


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


import test_gpu_oop_random as OR  # noqa: E402


# ------------------------------------------------------------------------------------------------ patterns and f
def pattern(m, n, lens, rng, *, sorted_=True, repeats=False):
    """(rowptr, cols), 0-based: row r holds lens[r] stored columns, ascending and distinct, or in random order, or (repeats)
    with repeated columns"""
    rows = []
    for k in lens:
        if repeats:
            c = rng.integers(0, n, k)
            if k > 1:
                c[rng.integers(0, k)] = c[0]
        else:
            c = rng.choice(n, min(k, n), replace=False)
            if sorted_:
                c = np.sort(c)
        rows.append(np.asarray(c, np.int64))
    lens = np.array([len(c) for c in rows], np.int64)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    cols = np.concatenate(rows) if len(rows) and lens.sum() else np.zeros(0, np.int64)
    return rp, cols


def ell_of(m, n, rp, cols, rng, K=3, zero_share=0.1):
    """the ELL rows function whose row r reads K of its stored columns (random ones when the row is empty), with about one
    coefficient in ten exactly 0: those entries' quotients are +-0 and dropped"""
    ec = np.empty((K, m), np.int64)
    for r in range(m):
        own = cols[rp[r]:rp[r + 1]]
        ec[:, r] = rng.choice(own, K) if len(own) else rng.integers(0, n, K)
    coef = rng.uniform(0.5, 2.0, (K, m)) * rng.choice([-1.0, 1.0], (K, m))
    coef[rng.random((K, m)) < zero_share] = 0.0
    return OR.Ell(ec, coef)


def csc_of_entry_set(m, n, rp, cols):
    A = sps.csr_matrix((np.ones(len(cols)), cols, rp), shape=(m, n)).tocsc()
    A.sum_duplicates()
    A.sort_indices()
    return A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1


def csr_mirror(pkg, m, n, rp, cols):
    return pkg.SparseMatrixCSR(m, n, torch.from_numpy(rp + 1), torch.from_numpy(cols + 1),
                               torch.zeros(len(cols), dtype=torch.float64, device="cuda"))


def expected_csr(res_csc, m, n, rp, cols):
    """the CSC result's kept values at the CSR sparsity's slots, in slot order: (rowptr, colval, nzval), 1-based"""
    cp = res_csc.colptr.cpu().numpy() - 1
    rv = res_csc.rowval.cpu().numpy() - 1
    nz = res_csc.nzval.cpu().numpy()
    cc = np.repeat(np.arange(n, dtype=np.int64), np.diff(cp))
    keys = rv * n + cc
    o = np.argsort(keys, kind="stable")
    keys, nz = keys[o], nz[o]
    srow = np.repeat(np.arange(m, dtype=np.int64), np.diff(rp))
    skey = srow * n + cols
    i = np.searchsorted(keys, skey)
    present = i < len(keys)
    present[present] = keys[i[present]] == skey[present]
    rowptr = 1 + np.concatenate([[0], np.cumsum(np.bincount(srow[present], minlength=m))]).astype(np.int64)
    return rowptr, cols[present] + 1, nz[i[present]]


def assert_csr(got, want, m, n, what):
    assert type(got).__name__ == "SparseMatrixCSR", what
    assert got.shape == (m, n), what
    assert np.array_equal(got.rowptr.cpu().numpy(), want[0]), f"{what}: rowptr"
    assert np.array_equal(got.colval.cpu().numpy(), want[1]), f"{what}: colval"
    assert got.nnz == len(want[1]), f"{what}: kept count"
    assert_same_bits(got.nzval.cpu().numpy(), want[2], f"{what}: nzval")


def run_case(pkg, oracle, ell, x, rp, cols, cv, *, fd="forward", dir=1.0, steps=(None, None), f_in=False, max_batch=1,
             scratch=0, sm=None, what=""):
    """(CSR result, CSR plan, CSC result, CSC plan): the CSC route held to the oracle, the CSR route held to it"""
    m, n = ell.m, len(x)
    cp, rv = csc_of_entry_set(m, n, rp, cols)
    res_csc, plan_csc = OR.run_csc(pkg, oracle, ell, x, cp, rv, cv, fd=fd, sparse=True, dir=dir, steps=steps, f_in=f_in,
                                   max_batch=max_batch, scratch=scratch, sm=sm, what=what)
    complex_ = fd == "complex"
    f, ctx = ell.native(pkg, complex_)
    xd = torch.from_numpy(x.copy()).cuda()
    fin = torch.from_numpy(OR.Twin(ell, oracle)(x)).cuda() if f_in else None
    kw = {"max_batch": max_batch}
    if scratch:
        kw["scratch_bytes"] = scratch
    cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd, **kw)
    M = csr_mirror(pkg, m, n, rp, cols)
    skw = {} if complex_ else {"relstep": steps[0], "absstep": steps[1], "dir": dir}
    with fdb_env(SM_COUNT=sm):
        res = pkg.finite_difference_jacobian(f, xd, cache, fin, colorvec=cv, sparsity=M, jac_prototype=M.similar(), **skw)
        torch.cuda.synchronize()
    plan = cache._last_plan
    Cn = max(int(cv.max(initial=0)), 0)
    calls = 2 * Cn if fd == "central" else Cn + (1 if fd == "forward" and not f_in else 0)
    assert ctx.calls == calls, f"{what}: {ctx.calls} calls, expected {calls}"
    info = plan.info()
    assert info["n_entries"] == len(cols) and info["jkind"] == pkg._lib.FDB_J_CSR, what
    if not complex_ and Cn > 0:
        assert_same_bits(np.asarray(plan.eps()[:Cn]), np.asarray(plan_csc.eps()[:Cn]), f"{what}: step sizes")
    assert_csr(res, expected_csr(res_csc, m, n, rp, cols), m, n, what)
    return res, plan, res_csc, plan_csc


def random_case(seed, m=None, n=None, *, sorted_=True, repeats=False, empty_share=0.2, maxlen=7):
    rng = np.random.default_rng(seed)
    m = int(rng.integers(1, 600)) if m is None else m
    n = int(rng.integers(1, 600)) if n is None else n
    lens = rng.integers(0, maxlen, m)
    lens[rng.random(m) < empty_share] = 0
    rp, cols = pattern(m, n, lens, rng, sorted_=sorted_, repeats=repeats)
    ell = ell_of(m, n, rp, cols, rng)
    x = OR.make_x(rng, n)
    return rng, ell, x, rp, cols


def colouring(kind, rng, m, n, rp, cols):
    cp, rv = csc_of_entry_set(m, n, rp, cols)
    if kind == "matrix_colors":
        return OR.greedy_colouring(m, n, cp, rv, rng)
    if kind == "random":
        return rng.integers(1, 6, n).astype(np.int64)
    if kind == "colourless":
        cv = OR.greedy_colouring(m, n, cp, rv, rng)
        cv[rng.random(n) < 0.3] = 0
        return cv
    return np.zeros(n, np.int64)                                         # "none"


# ------------------------------------------------------------------------------------------------ patterns x colourings
@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
@pytest.mark.parametrize("shape", ["sorted", "unsorted", "repeated", "m_ne_n"])
def test_patterns_and_colourings(pkg, oracle, fd, shape):
    for i, cvk in enumerate(("matrix_colors", "random", "colourless", "none")):
        seed = 100 * i + len(shape)
        kw = {"sorted_": shape != "unsorted", "repeats": shape == "repeated"}
        if shape == "m_ne_n":
            rng, ell, x, rp, cols = random_case(seed, 350, 90, **kw)
        else:
            rng, ell, x, rp, cols = random_case(seed, **kw)
        cv = colouring(cvk, rng, ell.m, len(x), rp, cols)
        run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, what=f"{shape} {cvk} {fd}")


def test_sorted_rows_equal_the_csc_result_converted(pkg, oracle):
    """rows of sorted, distinct columns: the CSR result is exactly the CSC route's result converted to CSR"""
    rng, ell, x, rp, cols = random_case(5, 700, 500)
    cv = colouring("matrix_colors", rng, ell.m, len(x), rp, cols)
    res, _, res_csc, _ = run_case(pkg, oracle, ell, x, rp, cols, cv, what="sorted")
    h = sps.csc_matrix((res_csc.nzval.cpu().numpy(), res_csc.rowval.cpu().numpy() - 1, res_csc.colptr.cpu().numpy() - 1),
                       shape=res_csc.shape).tocsr()
    assert np.array_equal(res.rowptr.cpu().numpy(), h.indptr + 1)
    assert np.array_equal(res.colval.cpu().numpy(), h.indices + 1)
    assert_same_bits(res.nzval.cpu().numpy(), h.data, "values")


def test_empty_rows_long_rows_and_empty_runs(pkg, oracle):
    rng = np.random.default_rng(8)
    n = 3000
    cases = {
        "empty rows": np.where(rng.random(900) < 0.5, 0, rng.integers(1, 5, 900)),
        "run of 3000 empty rows": np.concatenate([[600], np.zeros(3000, np.int64), [700], np.zeros(1500, np.int64), [900]]),
        "row of 2600 entries": np.array([3, 0, 2600, 1, 0, 5]),
    }
    for name, lens in cases.items():
        m = len(lens)
        rp, cols = pattern(m, n, lens, rng, sorted_=False)
        ell = ell_of(m, n, rp, cols, rng)
        x = OR.make_x(rng, n)
        for fd in ("forward", "central"):
            cv = colouring("matrix_colors", rng, m, n, rp, cols)
            run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, sm=1, what=f"{name} {fd}")


def test_many_colours(pkg, oracle):
    """more than 8 colours (list-based step sizes, bit-equal to the CSC plan's) and more than 1024 colours"""
    rng = np.random.default_rng(21)
    for m, n, C_ in ((400, 300, 40), (1500, 1400, 1300)):
        lens = rng.integers(0, 5, m)
        rp, cols = pattern(m, n, lens, rng, sorted_=False)
        ell = ell_of(m, n, rp, cols, rng)
        x = OR.make_x(rng, n)
        cv = rng.permutation(np.arange(n) % C_ + 1).astype(np.int64)
        for fd in ("forward", "central"):
            _, plan, _, _ = run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, max_batch=64, what=f"C={C_} {fd}")
            assert plan.info()["n_colors"] == C_


@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("dir,steps,f_in", [(-1.0, (None, None), True), (0.3, (1e-4, None), False),
                                            (1.0, (None, 1e-3), True), (-1.0, (1e-5, 0.0), False)])
def test_step_options(pkg, oracle, fd, dir, steps, f_in):
    rng, ell, x, rp, cols = random_case(33, 500, 400, sorted_=False)
    cv = colouring("colourless", rng, ell.m, len(x), rp, cols)
    run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, dir=dir, steps=steps, f_in=f_in and fd == "forward",
             what=f"dir={dir} steps={steps}")


@pytest.mark.parametrize("E", [1021, 1022, 1023, 1024, 1025, 1026, 1027, 1028, 1029, 2047, 2048, 2049])
def test_tile_edges_on_one_sm(pkg, oracle, E):
    """candidate counts around one and two tiles with one SM: blocks loop over tiles and the look-back crosses them"""
    rng = np.random.default_rng(E)
    m = E // 3
    lens = np.full(m, 3, np.int64)
    lens[: E - 3 * m] += 1
    lens[rng.permutation(m)[: m // 5]] = 0
    lens[0] += E - lens.sum()
    rp, cols = pattern(m, 60, lens, rng, repeats=True)
    assert len(cols) == E
    ell = ell_of(m, 60, rp, cols, rng)
    x = OR.make_x(rng, 60)
    for fd in ("forward", "central"):
        cv = colouring("random", rng, m, 60, rp, cols)
        run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, sm=1, what=f"E={E} {fd}")


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_copy_path_equals_fused(pkg, oracle, fd):
    """one f! output per group (the CSR scatter writes the candidates, the compaction copies them) against the fused
    compaction on the same problem"""
    rng, ell, x, rp, cols = random_case(44, 800, 600, sorted_=False)
    cv = colouring("colourless", rng, ell.m, len(x), rp, cols)
    fused, pf, _, _ = run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, max_batch=64, what=f"fused {fd}")
    scratch = 8 * (ell.m + 2) * (2 if fd == "central" else 1) + 64
    copy, pc, _, _ = run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, max_batch=1, scratch=scratch, what=f"copy {fd}")
    assert pf.info()["n_groups"] == 1 and pc.info()["n_groups"] > 1
    assert torch.equal(fused.rowptr, copy.rowptr) and torch.equal(fused.colval, copy.colval)
    assert torch.equal(fused.nzval.view(torch.int64), copy.nzval.view(torch.int64))


@pytest.mark.parametrize("fd", ["forward", "central"])
def test_ieee_edges(pkg, oracle, fd):
    """x with NaN and +-Inf gives NaN quotients (kept), zero coefficients +0.0 / -0.0 ones (dropped)"""
    rng, ell, x, rp, cols = random_case(55, 400, 300, sorted_=False)
    x[rng.integers(0, 300, 4)] = [np.nan, np.inf, -np.inf, np.nan]
    cv = colouring("matrix_colors", rng, ell.m, len(x), rp, cols)
    for dir in (1.0, -1.0):
        res, _, _, _ = run_case(pkg, oracle, ell, x, rp, cols, cv, fd=fd, dir=dir, what=f"ieee {fd} dir={dir}")
        v = res.nzval.cpu().numpy()
        assert np.isnan(v).any() and not (v == 0.0).any()


# ------------------------------------------------------------------------------------------------ through Python f
def _recording(ell):
    def f(x):
        f.points.append(x.detach().cpu().numpy().copy())
        return ell.torch_f(x)
    f.points = []
    return f


@pytest.mark.parametrize("fd", ["forward", "central"])
def test_points_and_cacheless_form(pkg, fd):
    """the points f sees, and their order, equal the CSC route's; the cache-less form gives the cached form's result"""
    rng, ell, x, rp, cols = random_case(66, 300, 250, sorted_=False)
    m, n = ell.m, len(x)
    cv = colouring("colourless", rng, m, n, rp, cols)
    cp, rv = csc_of_entry_set(m, n, rp, cols)
    xd = torch.from_numpy(x).cuda()
    M = csr_mirror(pkg, m, n, rp, cols)
    S = pkg.SparseMatrixCSC(m, n, torch.from_numpy(cp), torch.from_numpy(rv), None)
    out = {}
    for name, sp, proto in (("csr", M, M.similar()), ("csc", S, S), ("csc->csr", S, M.similar())):
        f = _recording(ell)
        cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd)
        r = pkg.finite_difference_jacobian(f, xd, cache, colorvec=cv, sparsity=sp, jac_prototype=proto, dir=-1.0)
        r2 = pkg.finite_difference_jacobian(f, xd, cache, colorvec=cv, sparsity=sp, jac_prototype=proto, dir=-1.0)
        out[name] = (r, f.points, r2)
    assert len(out["csr"][1]) == len(out["csc"][1]) == len(out["csc->csr"][1])
    for a, b, c in zip(out["csr"][1], out["csc"][1], out["csc->csr"][1]):
        assert_same_bits(a, b, "points")
        assert_same_bits(a, c, "points")
    want = expected_csr(out["csc"][0], m, n, rp, cols)
    assert_csr(out["csr"][0], want, m, n, "csr")
    assert_csr(out["csr"][2], want, m, n, "csr, plan reused")
    # a CSC sparsity with a CSR prototype: the CSR of its entry set (sorted rows)
    A = sps.csc_matrix((np.ones(len(rv)), rv - 1, cp - 1), shape=(m, n)).tocsr()
    assert_csr(out["csc->csr"][0], expected_csr(out["csc"][0], m, n, A.indptr.astype(np.int64),
                                                A.indices.astype(np.int64)), m, n, "csc sparsity")
    cl = pkg.finite_difference_jacobian(ell.torch_f, xd, fd, colorvec=cv, sparsity=M, jac_prototype=M.similar(), dir=-1.0)
    assert_csr(cl, want, m, n, "cache-less")


def test_empty_shapes(pkg):
    """m = 0 and nnz = 0: a row pointer of ones and no entry"""
    for m, n, lens in ((0, 5, []), (4, 6, [0, 0, 0, 0])):
        rp = np.concatenate([[0], np.cumsum(np.asarray(lens, np.int64))]).astype(np.int64)
        cols = np.zeros(0, np.int64)
        M = csr_mirror(pkg, m, n, rp, cols)
        x = torch.linspace(-1, 1, n, dtype=torch.float64, device="cuda")
        for fd in ("forward", "central"):
            r = pkg.finite_difference_jacobian(lambda v: v[:m] * 2.0, x, fd, sparsity=M, jac_prototype=M.similar())
            assert r.shape == (m, n) and r.nnz == 0
            assert np.array_equal(r.rowptr.cpu().numpy(), np.ones(m + 1, np.int64))


# ------------------------------------------------------------------------------------------------ groups
def _group(pkg, fdist, devs, fd, sp, proto, cv, ell, x, **kw):
    g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=sp, jac_prototype=proto, **kw)
    fs = [_recording(ell) for _ in devs]
    try:
        res = g.run(fs, x)
        torch.cuda.synchronize()
        return res, sum(len(f.points) for f in fs)
    finally:
        g.close()


def _same(a, b, what):
    assert type(a).__name__ == type(b).__name__ == "SparseMatrixCSR", what
    assert torch.equal(a.rowptr, b.rowptr) and torch.equal(a.colval, b.colval), what
    assert torch.equal(a.nzval.view(torch.int64), b.nzval.view(torch.int64)), what


@pytest.mark.parametrize("fd", ["forward", "central"])
def test_groups_match_one_device(pkg, fdist, fd):
    rng, ell, x, rp, cols = random_case(77, 600, 500, sorted_=False)
    m, n = ell.m, len(x)
    xd = torch.from_numpy(x).cuda()
    M = csr_mirror(pkg, m, n, rp, cols)
    sets = [[0, 0], [0, 0, 0], [0, 0, 0, 0]]
    if torch.cuda.device_count() >= 2:
        sets += [[0, 1], [1, 0, 1]]
    for cvk in ("colourless", "few"):
        cv = colouring("colourless", rng, m, n, rp, cols) if cvk == "colourless" else \
            np.where(np.arange(n) % 2 == 0, 1, 2).astype(np.int64)           # C = 2 < world for 3 and 4 members
        single = pkg.finite_difference_jacobian(_recording(ell), xd, pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64,
                                                device="cuda"), fd), colorvec=cv, sparsity=M, jac_prototype=M.similar())
        want, calls = _group(pkg, fdist, [0], fd, M, M.similar(), cv, ell, xd)
        _same(want, single, "group [0]")
        for devs in sets:
            for part in (0, 1):
                got, gcalls = _group(pkg, fdist, devs, fd, M, M.similar(), cv, ell, xd, partition=part)
                assert gcalls == calls, devs
                _same(got, want, f"{devs} partition={part} {cvk}")
    # a CSC sparsity with a CSR prototype, in a group
    cp, rv = csc_of_entry_set(m, n, rp, cols)
    S = pkg.SparseMatrixCSC(m, n, torch.from_numpy(cp), torch.from_numpy(rv), None)
    got, _ = _group(pkg, fdist, [0, 0], fd, S, M.similar(), cv, ell, xd)
    one = pkg.finite_difference_jacobian(_recording(ell), xd, fd, colorvec=cv, sparsity=S, jac_prototype=M.similar())
    _same(got, one, "csc sparsity group")


def test_graph_replay_after_x_changes(pkg, fdist):
    rng, ell, x, rp, cols = random_case(88, 400, 300, sorted_=False)
    m, n = ell.m, len(x)
    M = csr_mirror(pkg, m, n, rp, cols)
    cv = colouring("matrix_colors", rng, m, n, rp, cols)
    xd = torch.from_numpy(x).cuda()
    g = fdist.GroupJacobianOOP([0], "forward", colorvec=cv, sparsity=M, jac_prototype=M.similar(), use_graph=True)
    try:
        f = ell.torch_f                             # no host copy: the call is captured into a graph
        g.run([f], xd)
        xd.mul_(1.5).add_(0.25)                     # x changes in place: the same buffers, the next call replays
        got = g.run([f], xd)
        torch.cuda.synchronize()
    finally:
        g.close()
    want = pkg.finite_difference_jacobian(_recording(ell), xd, "forward", colorvec=cv, sparsity=M, jac_prototype=M.similar())
    _same(got, want, "graph replay")


def test_complex_group_refused_before_any_f_call(pkg, fdist):
    rng, ell, x, rp, cols = random_case(99, 50, 40)
    M = csr_mirror(pkg, ell.m, len(x), rp, cols)
    g = fdist.GroupJacobianOOP([0, 0], "complex", sparsity=M, jac_prototype=M.similar())
    f = _recording(ell)
    try:
        with pytest.raises(pkg._lib.FdbError):
            g.run([f, f], torch.from_numpy(x).cuda())
    finally:
        g.close()
    assert f.points == []


# ------------------------------------------------------------------------------------------------ the C ABI directly
def _create(pkg, m, n, rp1, cv1, cv, kind, **opt):
    L = pkg._lib
    from finitediff_jl_b200 import api
    o = api._opts(L.FDB_FORWARD, 0, **opt)
    h = C.c_void_p()
    st = L.lib().fdb_oop_plan_create_csr(C.byref(h), m, n, rp1.ctypes.data, cv1.ctypes.data if len(cv1) else None,
                                         cv.ctypes.data if cv is not None else None, kind, max(m, 1), C.byref(o))
    return st, h


def test_refusals(pkg):
    L = pkg._lib
    m = n = 64
    rp1 = np.arange(0, 3 * m + 1, 3, dtype=np.int64) + 1
    cv1 = (np.arange(3 * m) % n + 1).astype(np.int64)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    calls = []

    @L.FDB_FN
    def f(ctx, fx, x, batch, ldfx, ldx, stream):
        calls.append(1)
        return 0

    st, h = _create(pkg, m, n, rp1, cv1, cv, L.FDB_OOP_DENSE)
    assert st == L.FDB_ERR_UNSUPPORTED and not h.value and "not built" in L.lib().fdb_last_error().decode()
    st, h = _create(pkg, m, n, rp1, cv1, cv, L.FDB_OOP_RAW)
    assert st == L.FDB_ERR_INVALID and not h.value
    st, h = _create(pkg, m, 0, rp1, cv1, None, L.FDB_OOP_SPARSE)
    assert st == L.FDB_ERR_INVALID and not h.value
    bad = rp1.copy()
    bad[5] = bad[6] + 1
    st, h = _create(pkg, m, n, bad, cv1, cv, L.FDB_OOP_SPARSE)
    assert st == L.FDB_ERR_INVALID and not h.value and "row pointer" in L.lib().fdb_last_error().decode()
    badc = cv1.copy()
    badc[7] = n + 1
    st, h = _create(pkg, m, n, rp1, badc, cv, L.FDB_OOP_SPARSE)
    assert st == L.FDB_ERR_INVALID and not h.value
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    buf = [torch.empty(k, dtype=dt, device="cuda") for k, dt in ((m + 1, torch.int64), (3 * m, torch.int64),
                                                                 (3 * m, torch.float64), (1, torch.int64))]

    def out(cap=3 * m, null=None):
        o = L.OopOut()
        o.colptr, o.rowval, o.nzval, o.nnz = (None if i == null else b.data_ptr() for i, b in enumerate(buf))
        o.cap = cap
        return o

    def jac(h, o):
        return L.lib().fdb_jacobian_oop(h, f, None, x.data_ptr(), C.byref(o), None, None, float("nan"), float("nan"), 1.0,
                                        None)
    st, h = _create(pkg, m, n, rp1, cv1, cv, L.FDB_OOP_SPARSE)
    assert st == L.FDB_OK
    assert jac(h, out(cap=3 * m - 1)) == L.FDB_ERR_INVALID
    for null in range(4):
        assert jac(h, out(null=null)) == L.FDB_ERR_INVALID
    info = L.PlanInfo()
    L.check(L.lib().fdb_plan_info(h, C.byref(info)))
    assert info.jkind == L.FDB_J_CSR and info.n_entries == 3 * m
    assert L.lib().fdb_plan_set_peers(h, 0, None) == L.FDB_ERR_UNSUPPORTED
    L.lib().fdb_plan_destroy(h)
    st, h = _create(pkg, m, n, rp1, cv1, cv, L.FDB_OOP_SPARSE, rank=0, world=2)
    assert st == L.FDB_OK
    assert jac(h, out()) == L.FDB_ERR_INVALID
    assert "fdb_group_create_oop_" in L.lib().fdb_last_error().decode()
    L.lib().fdb_plan_destroy(h)
    assert calls == []


# ------------------------------------------------------------------------------------------------ C2 size
class _Tridiag:
    def __init__(self, pkg, N):
        L = pkg._lib
        self.ctx = L.TridiagCtx(N, 0)
        self.fn = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, self.ctx)


@pytest.mark.parametrize("fd", ["forward", "central"])
def test_c2_size(pkg, fd):
    """N = 10^7 tridiagonal, 3 cyclic colours: the whole CSR result against the CSC route's, converted to CSR on the
    device"""
    L = pkg._lib
    N = 10_000_000
    A = sps.diags([np.ones(N - 1), np.ones(N), np.ones(N - 1)], [-1, 0, 1], format="csr")
    A.sort_indices()
    cv = (np.arange(N) % 3 + 1).astype(np.int64)
    x = torch.empty(N, dtype=torch.float64, device="cuda")
    L.synth().fdbs_fill_x(x.data_ptr(), N, 0x5EED, None)
    M = pkg.SparseMatrixCSR(N, N, torch.from_numpy(A.indptr.astype(np.int64) + 1).cuda(),
                            torch.from_numpy(A.indices.astype(np.int64) + 1).cuda(), None)
    T = A.tocsc()
    S = pkg.SparseMatrixCSC(N, N, torch.from_numpy(T.indptr.astype(np.int64) + 1).cuda(),
                            torch.from_numpy(T.indices.astype(np.int64) + 1).cuda(), None)
    del A, T
    out = {}
    for name, sp, proto in (("csr", M, M), ("csc", S, S)):
        fn = _Tridiag(pkg, N)
        cache = pkg.JacobianCache(x, torch.zeros(N, dtype=torch.float64, device="cuda"), fd)
        out[name] = (pkg.finite_difference_jacobian(fn.fn, x, cache, colorvec=cv, sparsity=sp, jac_prototype=proto),
                     fn.ctx.calls)
        torch.cuda.synchronize()
    r, c = out["csr"][0], out["csc"][0]
    assert out["csr"][1] == out["csc"][1]
    cols = torch.repeat_interleave(torch.arange(N, device="cuda"), torch.diff(c.colptr))
    key = (c.rowval - 1) * N + cols
    o = torch.argsort(key)
    rows = (c.rowval - 1)[o]
    rowptr = torch.ones(N + 1, dtype=torch.int64, device="cuda")
    rowptr[1:] += torch.cumsum(torch.bincount(rows, minlength=N), 0)
    assert torch.equal(r.rowptr, rowptr)
    assert torch.equal(r.colval, cols[o] + 1)
    assert torch.equal(r.nzval.view(torch.int64), c.nzval[o].view(torch.int64))
