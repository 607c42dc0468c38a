"""The block out-of-place Jacobians on the device (fdb_oop_plan_create_block_banded / _block_dense and their group forms,
through finite_difference_jacobian and GroupJacobianOOP with a SparseMatrixCSC prototype) against the CSC route given the
CSC of the same entry set E: colptr, rowval, the nzval bits, nnz, the f calls and the points passed to f must be
identical.  The CSC route is held to oop_oracle/ bit for bit elsewhere; a second section holds the block routes to the
restatement directly, with an ELL f that reads exactly E, and to the analytic derivative.  Last: one BlockSkylineMatrix
block of 46 341 columns, 2 147 488 281 candidates, past 2^31."""
import ctypes as C

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


import test_gpu_oop_random as OR  # noqa: E402
from test_gpu_oop_banded import assert_same, assert_same_tuple, host, make_f, sparse_proto  # noqa: E402
from test_gpu_structured_fill import analytic_tolerance, ell_derivative  # noqa: E402


def entries(sp):
    """(rows, cols), 0-based, of findstructralnz in CSC order"""
    r, c, _ = sp.findstructralnz()
    o = np.lexsort((r, c))
    return r[o] - 1, c[o] - 1


def csc_of(pkg, sp):
    r, c = entries(sp)
    n = sp.shape[1]
    cp = np.concatenate([[0], np.cumsum(np.bincount(c, minlength=n))]).astype(np.int64) + 1
    return cp, (r + 1).astype(np.int64)


def csc_sparsity(pkg, sp):
    cp, rv = csc_of(pkg, sp)
    return pkg.SparseMatrixCSC(sp.shape[0], sp.shape[1], torch.from_numpy(cp), torch.from_numpy(rv), None)


def bbb(pkg, rb, l, u, lam, mu):
    return pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu))


def bsk(pkg, rb, l, u):
    return pkg.BlockSkylineMatrix(rb, rb, (l, u))


def _x(n, seed=0, edges=False):
    x = np.random.default_rng(seed).uniform(-1.5, 1.5, n)
    if n > 3:
        x[1], x[2] = -0.0, 0.0
    if edges and n > 8:
        x[4], x[5], x[6] = np.nan, np.inf, -np.inf
    return torch.from_numpy(x).cuda()


def run_pair(pkg, sp, fd, cv, *, dir=1.0, relstep=None, absstep=None, f_in=False, seed=0, edges=False, sm=None,
             **plan_kw):
    """(block result, CSC result, block plan); the f calls and the points each f saw are checked equal"""
    m, n = sp.shape
    x = _x(n, seed, edges)
    x0 = x.clone()
    out = []
    for which in ("block", "csc"):
        sparsity = sp if which == "block" else csc_sparsity(pkg, sp)
        f = make_f(m, n)
        cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device="cuda"), fd, **plan_kw)
        fin = f(x) if f_in else None
        f.points.clear()
        with fdb_env(SM_COUNT=sm):
            res = pkg.finite_difference_jacobian(f, x, cache, fin, relstep=relstep, absstep=absstep, dir=dir,
                                                 colorvec=cv, sparsity=sparsity, jac_prototype=sparse_proto(pkg, m, n))
            torch.cuda.synchronize()
        out.append((res, f.points, cache._last_plan))
        assert_same_bits(x.cpu().numpy(), x0.cpu().numpy(), "x modified")
    (rb, pb, planb), (rc, pc, planc) = out
    assert len(pb) == len(pc)
    for a, b in zip(pb, pc):
        assert_same_bits(a.view(np.float64), b.view(np.float64), "points f saw")
    assert planb.info()["n_entries"] == planc.info()["n_entries"] == len(entries(sp)[0])
    assert rb.nnz == rc.nnz
    return rb, rc, planb


def _types(pkg):
    """(name, block sparsity, its matrix_colors): non-uniform blocks, blocks of size 0 and 1, a large block beside small
    ones, sub-block bandwidths of a block or more, block bandwidths of nblocks or more"""
    out = [
        ("bbb uniform", bbb(pkg, [6] * 7, 1, 1, 1, 1)),
        ("bbb non-uniform, empty and size-1 blocks", bbb(pkg, [3, 0, 1, 7, 2, 5], 1, 2, 1, 0)),
        ("bbb large beside small", bbb(pkg, [40, 2, 1, 30, 3], 1, 1, 2, 1)),
        ("bbb lam, mu >= block", bbb(pkg, [4, 5, 3], 1, 0, 6, 9)),
        ("bbb l, u >= nblocks", bbb(pkg, [3, 4, 2], 5, 3, 0, 1)),
        ("padded BlockBandedMatrix", pkg.BlockBandedMatrix([4, 3, 5, 2], [4, 3, 5, 2], (1, 1))),
        ("skyline uniform", bsk(pkg, [5] * 8, 1, 1)),
        ("skyline non-uniform, empty and size-1 blocks", bsk(pkg, [3, 0, 1, 7, 2, 5], 2, 1)),
        ("skyline large beside small", bsk(pkg, [40, 2, 1, 30, 3], 1, 1)),
        ("skyline l, u >= nblocks", bsk(pkg, [3, 4, 2], 4, 6)),
    ]
    return [(name, sp, sp.matrix_colors()) for name, sp in out]


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_every_type_matches_the_csc_route(pkg, fd):
    for name, sp, cv in _types(pkg):
        rb, rc, plan = run_pair(pkg, sp, fd, cv)
        assert_same(rb, rc, f"{name} {fd}")


@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("dir,steps,f_in", [(-1.0, (None, None), True), (0.3, (1e-4, None), False),
                                            (1.0, (None, 1e-3), True), (-1.0, (1e-5, 0.0), False)])
def test_step_options_and_ieee_x_match(pkg, fd, dir, steps, f_in):
    for name, sp, cv in _types(pkg)[1::3]:
        rb, rc, _ = run_pair(pkg, sp, fd, cv, dir=dir, relstep=steps[0], absstep=steps[1], f_in=f_in and fd == "forward",
                             edges=True)
        assert_same(rb, rc, f"{name} {fd} dir={dir} steps={steps}")


def test_any_colouring(pkg):
    """table colourings (random, invalid, colour-less columns, none valid, identity) and the closed form"""
    sp_bb, sp_bd = bbb(pkg, [9, 4, 11, 6], 1, 1, 2, 1), bsk(pkg, [9, 4, 11, 6], 1, 1)
    for sp in (sp_bb, sp_bd):
        n = sp.shape[1]
        rng = np.random.default_rng(n)
        mc = sp.matrix_colors()
        colourings = {"matrix_colors": mc, "random invalid": rng.integers(1, 5, n),
                      "colour-less columns": np.where(rng.random(n) < 0.3, 0, mc), "none valid": np.zeros(n, np.int64),
                      "negative": -np.ones(n, np.int64), "identity": None}
        for fd in ("forward", "central", "complex"):
            for name, cv in colourings.items():
                cvv = range(1, n + 1) if cv is None else np.asarray(cv, np.int64)
                rb, rc, _ = run_pair(pkg, sp, fd, cvv)
                assert_same(rb, rc, f"{type(sp).__name__} {name} {fd}")


def test_closed_form_colouring_is_detected(pkg):
    """uniform blocks with matrix_colors read no colour table; the result is that of the same colours in a table"""
    for sp in (bbb(pkg, [7] * 9, 1, 1, 1, 1), bsk(pkg, [7] * 9, 1, 1)):
        cv = sp.matrix_colors()
        rb, rc, plan = run_pair(pkg, sp, "forward", cv)
        assert_same(rb, rc, type(sp).__name__)


def test_many_colours_and_wide_tables(pkg):
    """more than 1024 colours (16-bit table, list-based step sizes) and colour ids past 65535 (32-bit table)"""
    sp = bsk(pkg, [600, 500, 300], 1, 0)            # matrix_colors: 600 + 500 = 1100 colours
    cv = sp.matrix_colors()
    assert cv.max() == 1100
    for fd in ("forward", "central"):
        rb, rc, plan = run_pair(pkg, sp, fd, cv, max_batch=8)
        assert plan.info()["n_colors"] == 1100 and plan.info()["color_bits"] == 16
        assert_same(rb, rc, f"1100 colours {fd}")
    sp = bbb(pkg, [30, 20, 25], 1, 1, 2, 2)
    rng = np.random.default_rng(3)
    cv = OR.spread_ids(sp.matrix_colors(), 70_000, rng)
    for fd in ("forward", "complex"):
        rb, rc, plan = run_pair(pkg, sp, fd, cv, max_batch=8)
        assert plan.info()["color_bits"] == 32
        assert_same(rb, rc, f"32-bit {fd}")


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_candidate_copy_path(pkg, fd):
    """one f! output per group: the block scatter writes the candidates in the in-place layout and the compaction copies"""
    for sp in (bbb(pkg, [50, 30, 70, 10], 1, 1, 2, 3), bsk(pkg, [50, 30, 70, 10], 1, 1)):
        cv = sp.matrix_colors()
        cv[::9] = 0
        rb, rc, plan = run_pair(pkg, sp, fd, cv, max_batch=1, scratch_bytes=1)
        assert plan.info()["n_groups"] > 1
        assert_same(rb, rc, f"{type(sp).__name__} copy {fd}")


def tile_shapes(pkg):
    """(name, sparsity): candidate counts 1023, 1024, 1025, 2047 and 2049; their tiles cross block-column boundaries"""
    skyline = {1023: ([2] + [7] * 6 + [9], 1, 1), 1024: ([2] * 78 + [8], 1, 1), 1025: ([5] * 18 + [10], 1, 0),
               2047: ([9] * 13 + [2], 1, 0), 2049: ([5] * 41 + [3], 1, 0)}
    banded = {1023: [3] * 67 + [9], 1024: [3] * 66 + [17], 1025: [3] * 69, 2047: [3] * 135 + [11], 2049: [3] * 137 + [1]}
    out = []
    for E, (rb, l, u) in skyline.items():
        sp = bsk(pkg, rb, l, u)
        assert sp.j_len == E
        out.append((f"skyline E={E}", sp))
        sp = bbb(pkg, banded[E], 1, 1, 1, 0)
        assert len(sp.findstructralnz()[0]) == E
        out.append((f"bbb E={E}", sp))
    return out


@pytest.mark.parametrize("sm", [None, 1])
def test_tile_boundaries(pkg, sm):
    for name, sp in tile_shapes(pkg):
        for fd in ("forward", "central"):
            rb, rc, _ = run_pair(pkg, sp, fd, sp.matrix_colors(), sm=sm, dir=-1.0)
            assert_same(rb, rc, f"{name} sm={sm} {fd}")
    # block-dense tiles spanning more than 256 block columns (the unstaged search), then fewer
    sp = bsk(pkg, [1] * 1500 + [40] * 30, 1, 1)
    rb, rc, _ = run_pair(pkg, sp, "forward", sp.matrix_colors(), sm=sm)
    assert_same(rb, rc, f"staging switch sm={sm}")


def test_padded_block_banded_equals_skyline(pkg):
    """one structure in two storages, one colorvec: the same sparse result"""
    rb = [5, 3, 6, 4, 5]
    a, b = pkg.BlockBandedMatrix(rb, rb, (1, 1)), bsk(pkg, rb, 1, 1)
    assert np.array_equal(np.stack(entries(a)), np.stack(entries(b)))
    cv = b.matrix_colors()
    for fd in ("forward", "central", "complex"):
        x = _x(b.n, 4)
        res = []
        for sp in (a, b):
            f = make_f(b.n, b.n)
            cache = pkg.JacobianCache(x, fd)
            res.append(host(pkg.finite_difference_jacobian(f, x, cache, colorvec=cv, sparsity=sp,
                                                           jac_prototype=sparse_proto(pkg, b.n, b.n))))
        assert_same_tuple(res[0], res[1], fd)


def test_reused_plan_and_graph_replay(pkg, fdist):
    """a cached plan run on several x, and a group [0] capturing its call once and replaying it while x changes in place"""
    for sp in (bbb(pkg, [8] * 20, 1, 1, 1, 1), bsk(pkg, [8] * 20, 1, 1)):
        n = sp.shape[1]
        cv = sp.matrix_colors()
        ell = block_ell(sp, 5)
        f, _ = ell.native(pkg)
        xd = _x(n, 1)
        cache = pkg.JacobianCache(xd, "central")
        g = fdist.GroupJacobianOOP([0], "central", colorvec=cv, sparsity=sp, jac_prototype=sparse_proto(pkg, n, n),
                                   use_graph=True)
        try:
            for seed in (1, 2, 3):
                xd.copy_(_x(n, seed))
                got = pkg.finite_difference_jacobian(f, xd, cache, colorvec=cv, sparsity=sp,
                                                     jac_prototype=sparse_proto(pkg, n, n), dir=-1.0)
                replay = g.run([f], xd, dir=-1.0)
                fresh = pkg.finite_difference_jacobian(f, xd, pkg.JacobianCache(xd, "central"), colorvec=cv,
                                                       sparsity=csc_sparsity(pkg, sp),
                                                       jac_prototype=sparse_proto(pkg, n, n), dir=-1.0)
                torch.cuda.synchronize()
                assert_same(got, fresh, f"reused {seed}")
                assert_same_tuple(host(replay), host(fresh), f"replay {seed}")
            assert g.plans[0].counters()["jacobians"] == 3
        finally:
            g.close()


@pytest.mark.parametrize("fd", ["forward", "central"])
def test_groups_match_one_device(pkg, fdist, fd):
    for sp in (bbb(pkg, [20, 7, 0, 13, 9], 1, 2, 2, 1), bsk(pkg, [20, 7, 0, 13, 9], 2, 1)):
        n = sp.shape[1]
        for cv in (sp.matrix_colors(), np.where(np.arange(n) % 5 == 0, 0, sp.matrix_colors()), np.zeros(n, np.int64)):
            x = _x(n, 3)
            single = pkg.finite_difference_jacobian(make_f(n, n), x, pkg.JacobianCache(x, fd), colorvec=cv, sparsity=sp,
                                                    jac_prototype=sparse_proto(pkg, n, n))
            want = host(single)
            sets = [[0], [0, 0], [0, 0, 0]] + ([[0, 1]] if torch.cuda.device_count() >= 2 else [])
            for devs in sets:
                for partition in (0, 1):
                    g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=sp, jac_prototype=sparse_proto(pkg, n, n),
                                               partition=partition)
                    fs = [make_f(n, n) for _ in devs]
                    try:
                        got = host(g.run(fs, x))
                        torch.cuda.synchronize()
                    finally:
                        g.close()
                    assert_same_tuple(got, want, f"{type(sp).__name__} {devs} partition={partition}")


def test_stencil_g1000(pkg):
    """the 5-point Laplacian structure of a 1000 x 1000 grid: 1000 blocks of 1000, (l, u) = (1, 1), (lam, mu) = (1, 1);
    BandedBlockBandedMatrix's matrix_colors has 9 colours.  Held to the CSC route with a structure-reading f."""
    g = 1000
    sp = bbb(pkg, [g] * g, 1, 1, 1, 1)
    cv = sp.matrix_colors()
    assert cv.max() == 9
    ell = OR.Ell(*lap5_ell(g))                     # holds the device arrays f reads
    f, _ = ell.native(pkg)
    x = _x(g * g, 7)
    res = []
    for s in (sp, csc_sparsity(pkg, sp)):
        cache = pkg.JacobianCache(x, "forward")
        res.append(pkg.finite_difference_jacobian(f, x, cache, colorvec=cv, sparsity=s,
                                                  jac_prototype=sparse_proto(pkg, g * g, g * g)))
        torch.cuda.synchronize()
    assert cache._last_plan.info()["n_entries"] == len(entries(sp)[0])
    assert_same(res[0], res[1], "g=1000")


def lap5_ell(g):
    """(cols, coef) of f_i = 4 x_i - the grid neighbours of i inside a g x g grid (ELL, padding with coefficient 0)"""
    i = np.arange(g * g)
    r, c = i % g, i // g
    nb = [i, np.where(r > 0, i - 1, i), np.where(r < g - 1, i + 1, i), np.where(c > 0, i - g, i),
          np.where(c < g - 1, i + g, i)]
    coef = [np.full(g * g, 4.0), np.where(r > 0, -1.0, 0.0), np.where(r < g - 1, -1.0, 0.0), np.where(c > 0, -1.0, 0.0),
            np.where(c < g - 1, -1.0, 0.0)]
    return np.stack(nb).astype(np.int32), np.stack(coef)


def test_refusals_before_any_f_call(pkg):
    L = pkg._lib
    from finitediff_jl_b200 import api
    o = api._opts(L.FDB_FORWARD, 0)
    blocks = np.array([3, 4], np.int64)
    bp = blocks.ctypes.data
    cases = [
        ("bb dense result", "block_banded", (2, bp, 1, 1, 0, 0, None, L.FDB_OOP_DENSE, 7), L.FDB_ERR_UNSUPPORTED),
        ("bb raw result", "block_banded", (2, bp, 1, 1, 0, 0, None, L.FDB_OOP_RAW, 7), L.FDB_ERR_INVALID),
        ("bb negative l", "block_banded", (2, bp, -1, 1, 0, 0, None, L.FDB_OOP_SPARSE, 7), L.FDB_ERR_INVALID),
        ("bb negative mu", "block_banded", (2, bp, 1, 1, 0, -1, None, L.FDB_OOP_SPARSE, 7), L.FDB_ERR_INVALID),
        ("bb NULL blocks", "block_banded", (2, None, 1, 1, 0, 0, None, L.FDB_OOP_SPARSE, 7), L.FDB_ERR_INVALID),
        ("bb n = 0", "block_banded", (0, None, 1, 1, 0, 0, None, L.FDB_OOP_SPARSE, 1), L.FDB_ERR_INVALID),
        ("bd dense result", "block_dense", (2, bp, 1, 1, None, L.FDB_OOP_DENSE, 7), L.FDB_ERR_UNSUPPORTED),
        ("bd raw result", "block_dense", (2, bp, 1, 1, None, L.FDB_OOP_RAW, 7), L.FDB_ERR_INVALID),
        ("bd negative u", "block_dense", (2, bp, 1, -1, None, L.FDB_OOP_SPARSE, 7), L.FDB_ERR_INVALID),
        ("bd NULL blocks", "block_dense", (2, None, 1, 1, None, L.FDB_OOP_SPARSE, 7), L.FDB_ERR_INVALID),
        ("bd n = 0", "block_dense", (1, np.zeros(1, np.int64).ctypes.data, 1, 1, None, L.FDB_OOP_SPARSE, 1),
         L.FDB_ERR_INVALID),
    ]
    for name, suffix, args, want in cases:
        h = C.c_void_p()
        st = getattr(L.lib(), f"fdb_oop_plan_create_{suffix}")(C.byref(h), *args, C.byref(o))
        assert st == want and not h.value, (name, st)
    # the in-place creators' wording for the same refusals
    h = C.c_void_p()
    L.lib().fdb_oop_plan_create_block_banded(C.byref(h), 2, bp, -1, 1, 0, 0, None, L.FDB_OOP_SPARSE, 7, C.byref(o))
    oop_msg = L.lib().fdb_last_error()
    L.lib().fdb_plan_create_block_banded(C.byref(h), 2, bp, -1, 1, 0, 0, 1000, None, C.byref(o))
    assert L.lib().fdb_last_error() == oop_msg
    # the mirror: a dense result raises before f is called
    sp = bsk(pkg, [3, 4], 1, 1)
    f = make_f(7, 7)
    x = _x(7)
    with pytest.raises(TypeError):
        pkg.finite_difference_jacobian(f, x, pkg.JacobianCache(x, "central"), sparsity=sp)
    assert f.points == []
    # a sparse rank plan alone is refused by fdb_jacobian_oop, before any f call
    ow = api._opts(L.FDB_FORWARD, 0, rank=0, world=2)
    st = L.lib().fdb_oop_plan_create_block_dense(C.byref(h), 2, bp, 1, 1, None, L.FDB_OOP_SPARSE, 7, C.byref(ow))
    assert st == L.FDB_OK
    ell = block_ell(sp, 1)
    fn, ctx = ell.native(pkg)
    out = L.OopOut()
    cp = torch.empty(8, dtype=torch.int64, device="cuda")
    rv = torch.empty(64, dtype=torch.int64, device="cuda")
    nz = torch.empty(64, dtype=torch.float64, device="cuda")
    nnz = torch.empty(1, dtype=torch.int64, device="cuda")
    out.colptr, out.rowval, out.nzval, out.cap, out.nnz = cp.data_ptr(), rv.data_ptr(), nz.data_ptr(), 64, nnz.data_ptr()
    st = L.lib().fdb_jacobian_oop(h, C.c_void_p(fn.address), C.c_void_p(C.addressof(ctx)), x.data_ptr(), C.byref(out),
                                  None, None, float("nan"), float("nan"), 1.0, None)
    assert st == L.FDB_ERR_INVALID and ctx.calls == 0
    L.lib().fdb_plan_destroy(h)


# ---- held to the restatement (oop_oracle/) and the analytic derivative ----
def block_ell(sp, seed, zero_share=0.1):
    """row r reads exactly the columns of E in row r, in random order; coefficients +-[0.5, 2], about zero_share of them
    exactly 0"""
    m = sp.shape[0]
    r, c = entries(sp)
    rng = np.random.default_rng(seed)
    order = np.argsort(r, kind="stable")
    bounds = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=m))])
    K = int(np.diff(bounds).max())
    cols = np.zeros((K, m), np.int64)
    coef = np.zeros((K, m))
    for i in range(m):
        v = rng.permutation(c[order[bounds[i]:bounds[i + 1]]])
        cols[:, i] = v[0]
        cols[:len(v), i] = v
        a = rng.uniform(0.5, 2.0, len(v)) * np.where(rng.random(len(v)) < 0.5, -1.0, 1.0)
        a[rng.random(len(v)) < zero_share] = 0.0
        coef[:len(v), i] = a
    return OR.Ell(cols, coef)


def check_analytic(res, sp, ell, x, cv, eps, fd, what):
    """every kept entry is an entry of E of a coloured column, within the analytic tolerance of d f_r / d x_c; every
    dropped entry of a coloured column has a zero derivative"""
    cp, rv, nz = res.colptr.cpu().numpy(), res.rowval.cpu().numpy() - 1, res.nzval.cpu().numpy()
    cols = np.repeat(np.arange(len(cp) - 1), np.diff(cp))
    r, c = entries(sp)
    inE = set(zip(r.tolist(), c.tolist()))
    assert all((a, b) in inE for a, b in zip(rv.tolist(), cols.tolist())), f"{what}: an entry outside E"
    k = cv[cols] - 1
    assert np.all(k >= 0), f"{what}: an entry of a column without a colour"
    d, S, T = ell_derivative(ell.cols.astype(np.int64), ell.coef, rv, cols, x)
    tol = analytic_tolerance(fd, None if fd == "complex" else np.asarray(eps)[k], S, T, ell.K)
    bad = np.flatnonzero(~(np.abs(nz - d) <= tol))
    assert bad.size == 0, f"{what}: {bad.size} entries off the derivative"
    kept = set(zip(rv.tolist(), cols.tolist()))
    live = cv[c] > 0
    dropped = [(a, b) for a, b in zip(r[live].tolist(), c[live].tolist()) if (a, b) not in kept]
    if dropped:
        dr, dc = np.array(dropped).T
        dd, _, _ = ell_derivative(ell.cols.astype(np.int64), ell.coef, dr, dc, x)
        assert np.all(dd == 0), f"{what}: a dropped entry with a non-zero derivative"


def run_oracle(pkg, oracle, sp, cv, *, fd="forward", seed=0, analytic=True, **kw):
    ell = block_ell(sp, seed)
    x = np.random.default_rng(seed + 1).uniform(0.5, 1.5, sp.shape[1]) * np.where(
        np.random.default_rng(seed + 2).random(sp.shape[1]) < 0.5, -1.0, 1.0)
    cp, rv = csc_of(pkg, sp)
    res, plan = OR.run_csc(pkg, oracle, ell, x, cp, rv, cv, fd=fd, sparse=True, band=sp, **kw)
    assert plan.info()["n_entries"] == len(rv)
    if analytic and kw.get("steps", (None, None)) == (None, None) and kw.get("dir", 1.0) in (1.0, -1.0):
        check_analytic(res, sp, ell, x, cv, None if fd == "complex" else plan.eps(), fd, kw.get("what", ""))
    return res, plan


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_types_against_the_oracle(pkg, oracle, fd):
    for name, sp, cv in _types(pkg):
        run_oracle(pkg, oracle, sp, cv, fd=fd, seed=len(name), what=f"{name} {fd}")


OPTIONS = [("dir-", dict(dir=-1.0)), ("steps", dict(steps=(1e-5, 1e-9))), ("f_in", dict(f_in=True)),
           ("copy", dict(max_batch=1, scratch=1)), ("sm1", dict(sm=1))]


@pytest.mark.parametrize("opt", OPTIONS, ids=[o[0] for o in OPTIONS])
@pytest.mark.parametrize("fd", ["forward", "central"])
def test_options_against_the_oracle(pkg, oracle, opt, fd):
    name, kw = opt
    if kw.get("f_in") and fd != "forward":
        pytest.skip("f_in is the forward mode's f(x)")
    for sp in (bbb(pkg, [30, 12, 1, 25], 1, 1, 3, 2), bsk(pkg, [30, 12, 1, 25], 1, 2)):
        cv = sp.matrix_colors()
        cv[::11] = 0
        run_oracle(pkg, oracle, sp, cv, fd=fd, seed=17, what=f"{type(sp).__name__} {name} {fd}", **kw)


def test_many_colours_against_the_oracle(pkg, oracle):
    sp = bsk(pkg, [600, 500, 300], 1, 0)
    run_oracle(pkg, oracle, sp, sp.matrix_colors(), fd="central", seed=5, max_batch=8, record=False, native_twin=True,
               what="1100 colours")


@pytest.mark.parametrize("devs", [[0, 0], [0, 0, 0]], ids=["0-0", "0-0-0"])
def test_groups_against_the_oracle(pkg, oracle, fdist, devs):
    for sp in (bbb(pkg, [30, 12, 1, 25], 2, 1, 1, 2), bsk(pkg, [30, 12, 1, 25], 1, 1)):
        n = sp.shape[1]
        cv = sp.matrix_colors()
        cv[::7] = 0
        for fd in ("forward", "central"):
            single, plan = run_oracle(pkg, oracle, sp, cv, fd=fd, seed=91, record=False, what=f"{devs} {fd}")
            ell = block_ell(sp, 91)
            x = np.random.default_rng(92).uniform(0.5, 1.5, n) * np.where(np.random.default_rng(93).random(n) < 0.5,
                                                                          -1.0, 1.0)
            g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=sp, jac_prototype=sparse_proto(pkg, n, n))
            members = [ell.native(pkg) for _ in devs]
            try:
                res = g.run([f for f, _ in members], torch.from_numpy(x).cuda())
                torch.cuda.synchronize()
            finally:
                g.close()
            assert_same_tuple(host(res), host(single), f"{devs} {fd}")
            Cn = int(cv.max())
            assert sum(ctx.calls for _, ctx in members) == (2 * Cn if fd == "central" else Cn + 1)


# ---- past 2^31 candidates ----
def test_one_block_past_2_31(pkg):
    """one BlockSkylineMatrix block of 46 341 columns: 2 147 488 281 candidates, colorvec 1:n.  f is the C5 form
    (fdbs_rank1: f_i = x_i^2 + w_i S, S = sum(x) / n, O(n) per point), so no quotient is zero; the structure is checked
    exactly and sampled columns against d f_i / d x_c = 2 x_i [i = c] + w_i / n"""
    L = pkg._lib
    b = 46_341
    E = b * b
    assert E == 2_147_488_281 > 2 ** 31
    need = E * 8 * 3 + 10 * 2 ** 30              # candidates, rowval and nzval, and the colour loop's scratch
    free, _ = torch.cuda.mem_get_info()
    assert free >= need, f"the case needs {need / 2**30:.0f} GiB, {free / 2**30:.0f} GiB free"
    sp = pkg.BlockSkylineMatrix([b], [b], (0, 0), data=torch.zeros(1, dtype=torch.float64, device="cuda"))
    rng = np.random.default_rng(2)
    xs, ws = rng.uniform(0.5, 1.5, b), rng.uniform(0.5, 1.5, b)
    x, w = torch.from_numpy(xs).cuda(), torch.from_numpy(ws).cuda()
    bs = torch.zeros((b + 1023) // 1024, dtype=torch.float64, device="cuda")
    fn = pkg.NativeFn(C.cast(L.synth().fdbs_rank1, C.c_void_p).value, L.Rank1Ctx(b, w.data_ptr(), bs.data_ptr(), 1, 0))
    cache = pkg.JacobianCache(x, "forward")
    res = pkg.finite_difference_jacobian(fn, x, cache, colorvec=range(1, b + 1), sparsity=sp,
                                         jac_prototype=sparse_proto(pkg, b, b))
    torch.cuda.synchronize()
    plan = cache._last_plan
    assert plan.info()["n_entries"] == E
    assert res.nnz == E
    assert torch.equal(res.colptr, torch.arange(b + 1, dtype=torch.int64, device="cuda") * b + 1)
    ar = torch.arange(1, b + 1, dtype=torch.int64, device="cuda")
    for c0 in range(0, b, 1000):
        c1 = min(c0 + 1000, b)
        assert torch.equal(res.rowval[c0 * b:c1 * b].view(c1 - c0, b), ar.expand(c1 - c0, b)), c0
    eps = plan.eps()
    for c in (0, 1, 40_000, b - 1):                # the last columns' candidates lie past 2^31
        got = res.nzval[c * b:(c + 1) * b].cpu().numpy()
        d = ws / b
        d[c] += 2 * xs[c]
        tol = 4 * abs(eps[c]) + 64 * np.finfo(float).eps * 4 / abs(eps[c])
        assert np.all(np.abs(got - d) <= tol), (c, np.abs(got - d).max(), tol)
