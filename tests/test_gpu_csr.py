"""The CSR plan (fdb_plan_create_csr / fdb_group_create_csr): J is the nzval of a CSR matrix with the sparsity's pattern.
Every case is held bit for bit, with the same f-call count, to
  - the COO slot route (fdb_plan_create_coo, FDB_J_SLOTS, slots 1..nnz) on the same buffer,
  - the CSC route on the same matrix, its nzval permuted into CSR order, and
  - the CPU oracle given the device's step sizes (a CSR is a COO entry list with slots 1..nnz).
J is pre-filled with NaN (a sentinel where x itself holds NaN): the plan must write every slot."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, fdb_env  # noqa: E402

FD = {"forward": 0, "central": 1, "complex": 2}
DEV = torch.device("cuda:0")
SENT = -12345.678


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


def _csr(rp, cols, m, n):
    return sp.csr_matrix((np.ones(len(cols)), np.asarray(cols, np.int32), np.asarray(rp, np.int32)), shape=(m, n))


_ELL = {}


class _Ell:
    """fdbs_ellrows whose row i reads exactly the stored columns of CSR row i (a structure-filling f); about one
    coefficient in ten is exactly 0; padding repeats column 0 with coefficient 0."""

    def __init__(self, pkg, A, seed, complex_=False):
        L = pkg._lib
        key = (id(A), seed)
        if key not in _ELL:
            rng = np.random.default_rng(seed)
            m = A.shape[0]
            lens = np.diff(A.indptr)
            K = max(int(lens.max()) if m else 1, 1)
            rows = np.repeat(np.arange(m), lens)
            pos = np.arange(A.nnz) - A.indptr[rows]
            cols = np.zeros((K, m), np.int32)
            coef = np.zeros((K, m))
            v = rng.uniform(-1, 1, A.nnz)
            v[rng.random(A.nnz) < 0.1] = 0.0
            cols[pos, rows] = A.indices
            coef[pos, rows] = v
            _ELL[key] = (A, m, K, cols, coef, torch.from_numpy(cols).to(DEV), torch.from_numpy(coef).to(DEV))
        _, self.m, self.K, self.cols, self.coef, self.d_cols, self.d_coef = _ELL[key]
        self.ctx = L.EllCtx(self.m, self.K, self.d_cols.data_ptr(), self.d_coef.data_ptr(), 0)
        self.addr = C.cast(L.synth().fdbs_ellrows_c if complex_ else L.synth().fdbs_ellrows, C.c_void_p).value
        self.fn = pkg.NativeFn(self.addr, self.ctx)

    def oracle_ctx(self, oracle):
        return oracle.SynthEllCtx(self.m, self.K, self.cols.ctypes.data_as(C.POINTER(C.c_int32)),
                                  self.coef.ctypes.data_as(C.POINTER(C.c_double)), 1)


def _plan(api, creator, args, fdtype, keep, **opts):
    o = api._opts(FD[fdtype], 0, **opts)
    p = api.Plan(api._new_handle(f"fdb_plan_create_{creator}", *args, C.byref(o)).value)
    p._keep = keep
    return p


def _cvp(cv):
    return cv.ctypes.data if cv is not None and len(cv) else None


def _csr_plan(api, A, cv, fdtype, device_index=False, **opts):
    rp, cv_ = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    if device_index:
        rp, cv_ = torch.from_numpy(rp).to(DEV), torch.from_numpy(cv_).to(DEV)
        ptrs = (rp.data_ptr(), cv_.data_ptr() if A.nnz else None)
    else:
        ptrs = (rp.ctypes.data, cv_.ctypes.data if A.nnz else None)
    return _plan(api, "csr", (A.shape[0], A.shape[1], *ptrs, _cvp(cv)), fdtype, (rp, cv_, cv), **opts)


def _entries(A):
    coo = A.tocoo()
    return coo.row.astype(np.int64) + 1, coo.col.astype(np.int64) + 1, np.arange(1, A.nnz + 1, dtype=np.int64)


def _coo_plan(api, A, cv, fdtype, j_len=None, **opts):
    rows, cols, slots = _entries(A)
    return _plan(api, "coo", (A.shape[0], A.shape[1], A.nnz, rows.ctypes.data, cols.ctypes.data, api.L.FDB_J_SLOTS,
                              slots.ctypes.data, A.nnz if j_len is None else j_len, _cvp(cv)), fdtype,
                 (rows, cols, slots, cv), **opts)


def _csc_and_perm(A):
    """the CSC of A's stored entries (duplicates kept, rows ascending in a column) and, per CSC slot, its CSR slot"""
    T = sp.csr_matrix((np.arange(A.nnz, dtype=np.float64), A.indices, A.indptr), shape=A.shape).tocsc()
    return T.indptr.astype(np.int64) + 1, T.indices.astype(np.int64) + 1, T.data.astype(np.int64)


def _jac(pkg, plan, f, x, J, fdtype, relstep=None, absstep=None, dir=1.0, f_in=None):
    lib = pkg._lib.lib()
    ctx = C.addressof(f.ctx)
    Jp = J.data_ptr() if J.numel() else None
    if fdtype == "complex":
        st = lib.fdb_jacobian_complex(plan._h, f.addr, ctx, x.data_ptr() if x.numel() else None, Jp, None)
    else:
        st = lib.fdb_jacobian(plan._h, f.addr, ctx, x.data_ptr() if x.numel() else None, Jp, None,
                              None if f_in is None else f_in.data_ptr(), float("nan") if relstep is None else relstep,
                              float("nan") if absstep is None else absstep, float(dir), None)
    pkg._lib.check(st)
    torch.cuda.synchronize()


def _fin(pkg, A, x, seed):
    g = _Ell(pkg, A, seed)
    out = torch.empty(A.shape[0], dtype=torch.float64, device=DEV)
    assert pkg._lib.synth().fdbs_ellrows(C.addressof(g.ctx), out.data_ptr(), x.data_ptr(), 1, A.shape[0], A.shape[1], None) == 0
    torch.cuda.synchronize()
    return out


def _three(pkg, api, oracle, A, cv, fdtype, x, seed, kw, opts=None, sm=None):
    """CSR plan, COO slot route and CSC route (permuted) on one case; checks bits, f calls and the oracle."""
    opts = opts or {}
    cx = fdtype == "complex"
    m, n = A.shape
    f_in = _fin(pkg, A, x, seed) if kw.get("f_in") else None
    steps = {k: v for k, v in kw.items() if k != "f_in"}
    with fdb_env(SM_COUNT=sm):
        p_csr = _csr_plan(api, A, cv, fdtype, **opts)
        p_coo = _coo_plan(api, A, cv, fdtype, **opts)
    out = {}
    for name, plan in (("csr", p_csr), ("coo", p_coo)):
        f = _Ell(pkg, A, seed, cx)
        J = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
        _jac(pkg, plan, f, x, J, fdtype, f_in=f_in, **steps)
        out[name] = (J.cpu().numpy(), f.ctx.calls)
    what = f"{m}x{n} nnz={A.nnz} {fdtype} {kw} {opts}"
    info = p_csr.info()
    assert info["jkind"] == pkg._lib.FDB_J_CSR and info["n_entries"] == info["j_len"] == A.nnz, what
    assert info["alg_bytes_scatter"] == 32 * A.nnz + 16 * n + 8, what
    assert_same_bits(out["csr"][0], out["coo"][0], what + " vs COO", allow_nan=bool(np.isnan(x.cpu().numpy()).any()))
    assert out["csr"][1] == out["coo"][1] == info["fcalls_per_jacobian"] - (f_in is not None), what
    eps = p_csr.eps() if not cx else None
    if not cx:
        assert_same_bits(eps, p_coo.eps(), what + " steps")
    # the CSC route, permuted into CSR order (more than 8 colours: the CSC plan takes its steps from column lists, so it
    # is handed the CSR plan's steps)
    cp, rv, perm = _csc_and_perm(A)
    with fdb_env(SM_COUNT=sm):
        p_csc = _plan(api, "csc", (m, n, cp.ctypes.data, rv.ctypes.data if A.nnz else None, pkg._lib.FDB_J_CSC_NZVAL, None,
                                   None, 0, _cvp(cv)), fdtype, (cp, rv, cv), **opts)
    ext = None
    if not cx and info["n_colors"] > 8:
        ext = torch.from_numpy(eps).to(DEV)
        pkg._lib.check(pkg._lib.lib().fdb_plan_set_external_eps(p_csc._h, ext.data_ptr()))
    f = _Ell(pkg, A, seed, cx)
    Jc = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
    _jac(pkg, p_csc, f, x, Jc, fdtype, f_in=f_in, **steps)
    viacsc = np.empty(A.nnz)
    viacsc[perm] = Jc.cpu().numpy()
    assert_same_bits(out["csr"][0], viacsc, what + " vs CSC", allow_nan=True)
    assert f.ctx.calls == out["csr"][1], what
    # the oracle, fed the device's step sizes (its ELL f costs K*m per call: skipped where that makes hours of CPU time)
    if oracle is not None and _Ell(pkg, A, seed).K * m * (info["n_colors"] + 2) <= 3e8:
        rows, cols, slots = _entries(A)
        g = _Ell(pkg, A, seed)
        xh = x.cpu().numpy()
        ref = np.full(A.nnz, np.nan)
        okw = {}
        if f_in is not None:
            okw["f_in"] = f_in.cpu().numpy()
        if cx:
            r = oracle.jacobian_complex(oracle.Problem.coo_to_slots(m, n, rows, cols, slots, A.nnz), ref,
                                        oracle.native_fn("synth_ellrows_c"), xh, colorvec=cv, ctx=g.oracle_ctx(oracle))
        else:
            r = oracle.jacobian(oracle.Problem.coo_to_slots(m, n, rows, cols, slots, A.nnz), ref,
                                oracle.native_fn("synth_ellrows"), xh, fdtype=FD[fdtype], colorvec=cv, eps_override=eps,
                                ctx=g.oracle_ctx(oracle), dir=steps.get("dir", 1.0), **okw)
        assert_same_bits(out["csr"][0], ref, what + " vs oracle", allow_nan=True)
        assert r["fcalls"] == out["csr"][1], what
    return out["csr"][0]


def _valid_coloring(A, rng):
    T = A.tocsc()
    cv = np.zeros(A.shape[1], np.int64)
    for c in rng.permutation(A.shape[1]):
        rows = T.indices[T.indptr[c]:T.indptr[c + 1]]
        used = {int(cv[o]) for r in rows for o in A.indices[A.indptr[r]:A.indptr[r + 1]] if cv[o] > 0}
        k = 1
        while k in used:
            k += 1
        cv[c] = k
    return cv


def _patterns():
    rng = np.random.default_rng(3)
    out = {}
    m, n = 700, 600
    lens = rng.integers(0, 7, m)
    lens[rng.random(m) < 0.25] = 0
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["random_unsorted"] = _csr(rp, np.concatenate([rng.permutation(n)[:k] for k in lens]), m, n)
    lens = np.array([0, 2600, 1, 0, 0, 1500, 4, 1100, 0])
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["long_rows"] = _csr(rp, np.concatenate([rng.permutation(3000)[:k] for k in lens]), 9, 3000)
    lens = rng.integers(1, 6, 300)
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["repeated"] = _csr(rp, np.concatenate([np.full(k, rng.integers(0, 40)) if i % 3 == 0 else rng.integers(0, 40, k)
                                               for i, k in enumerate(lens)]), 300, 40)
    lens = np.zeros(12000, np.int64)
    lens[::4000] = 1500
    lens[-1] = 2
    rp = np.concatenate([[0], np.cumsum(lens)])
    out["empty_runs"] = _csr(rp, np.concatenate([rng.permutation(1600)[:k] for k in lens]), 12000, 1600)
    out["tall"] = _csr(*_band_csr(900, 300))
    out["nnz0"] = _csr(np.zeros(5, np.int64), np.zeros(0, np.int64), 4, 3)
    return out


def _band_csr(m, n):
    A = sp.diags([np.ones(n)] * 3, [-1, 0, 1], shape=(m, n), format="csr")
    A.sort_indices()
    return A.indptr, A.indices, m, n


PATTERNS = _patterns()


def _runs(fdtype):
    runs = [{}]
    if fdtype != "complex":
        runs += [{"relstep": 1e-5, "absstep": 1e-9}]
    if fdtype == "forward":
        runs += [{"dir": -1.0}, {"f_in": True}]
    return runs


@pytest.mark.parametrize("name", sorted(PATTERNS))
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_matches_coo_csc_and_oracle(pkg, api, oracle, name, fdtype):
    A = PATTERNS[name]
    m, n = A.shape
    rng = np.random.default_rng(len(name) + FD[fdtype])
    x = torch.from_numpy(rng.uniform(-2, 2, n)).to(DEV)
    valid = _valid_coloring(A, rng) if n else np.zeros(0, np.int64)
    cvs = {"valid": valid, "identity": np.arange(1, n + 1, dtype=np.int64)}
    if n > 2:
        inval = valid.copy()
        inval[rng.random(n) < 0.3] = 0          # colour-less columns
        inval[0] = -3
        cvs["colourless"] = inval
        cvs["invalid"] = (np.arange(n) % 2 + 1).astype(np.int64)      # two colours: rows collide
        cvs["cyclic"] = (np.arange(n) % max(int(valid.max()), 1) + 1).astype(np.int64)
    for cname, cv in cvs.items():
        for kw in _runs(fdtype) if cname == "valid" else [{}]:     # the step options once, on the valid colouring
            _three(pkg, api, oracle, A, cv, fdtype, x, 7, kw)


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_wide_tables_many_colours_and_multi_tile(pkg, api, oracle, fdtype):
    """8-, 16- and 32-bit colour tables, more than 1024 colours (global tables), FDB_SM_COUNT=1 (every block walks many
    tiles), several slab groups from a small scratch budget, and max_batch > 1."""
    A = PATTERNS["random_unsorted"]
    n = A.shape[1]
    x = torch.from_numpy(np.random.default_rng(9).uniform(-2, 2, n)).to(DEV)
    ident = np.arange(1, n + 1, dtype=np.int64)
    for cv in (ident, ident + 300, ident * 130):            # 600 colours (16 bit), 900, 78000 colours (32 bit)
        _three(pkg, api, None, A, cv, fdtype, x, 5, {}, sm=1)
    small = _valid_coloring(A, np.random.default_rng(1))
    for opts in ({"scratch_bytes": 8 * 704 * 3}, {"max_batch": 4}, {"scratch_bytes": 8 * 704 * 2, "max_batch": 2}):
        if fdtype == "complex" and "scratch_bytes" in opts:
            opts = dict(opts, scratch_bytes=2 * opts["scratch_bytes"])
        _three(pkg, api, oracle, A, small, fdtype, x, 5, {}, opts=opts, sm=1)
    B = PATTERNS["long_rows"]
    xb = torch.from_numpy(np.random.default_rng(2).uniform(-2, 2, B.shape[1])).to(DEV)
    _three(pkg, api, None, B, np.arange(1, B.shape[1] + 1, dtype=np.int64), fdtype, xb, 5, {}, sm=1)


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_ieee_edges(pkg, api, oracle, fdtype):
    A = PATTERNS["tall"]
    n = A.shape[1]
    xs = np.random.default_rng(4).uniform(-2, 2, n)
    xs[[0, 3, 5, 7, 9, 11, 13]] = [0.0, -0.0, np.nan, np.inf, -np.inf, -0.0, 1e300]
    x = torch.from_numpy(xs).to(DEV)
    for cv in ((np.arange(n) % 3 + 1).astype(np.int64), np.arange(1, n + 1, dtype=np.int64)):
        for kw in _runs(fdtype):
            _three(pkg, api, oracle, A, cv, fdtype, x, 11, kw)


def test_every_slot_written_and_tail_untouched(pkg, api):
    A = PATTERNS["empty_runs"]
    n = A.shape[1]
    x = torch.from_numpy(np.random.default_rng(6).uniform(-2, 2, n)).to(DEV)
    cv = _valid_coloring(A, np.random.default_rng(6))
    cv[::7] = 0
    for fdtype in ("forward", "central"):
        J = torch.full((A.nnz + 100,), SENT, dtype=torch.float64, device=DEV)
        J[: A.nnz] = float("nan")
        _jac(pkg, _csr_plan(api, A, cv, fdtype, device_index=True), _Ell(pkg, A, 1), x, J, fdtype)
        h = J.cpu().numpy()
        assert not np.isnan(h[: A.nnz]).any()
        assert (h[A.nnz:] == SENT).all()
        Jo = torch.full((A.nnz + 100,), SENT, dtype=torch.float64, device=DEV)
        _jac(pkg, _coo_plan(api, A, cv, fdtype, j_len=A.nnz + 100), _Ell(pkg, A, 1), x, Jo, fdtype)
        assert_same_bits(h[: A.nnz], Jo.cpu().numpy()[: A.nnz], f"{fdtype} long buffer", allow_nan=False)


def test_edge_sizes(pkg, api):
    """m = 0, n = 0 and nnz = 0: nothing to write, the f calls of the COO route."""
    for m, n in ((0, 4), (5, 0), (3, 3)):
        A = _csr(np.zeros(m + 1, np.int64), np.zeros(0, np.int64), m, n)
        for fdtype in ("forward", "central"):
            calls = []
            for route in (_csr_plan, _coo_plan):
                p = route(api, A, None, fdtype)
                x = torch.zeros(max(n, 1), dtype=torch.float64, device=DEV)
                fx = torch.zeros(max(m, 1), dtype=torch.float64, device=DEV)
                count = [0]

                def f(out, xx, count=count):
                    count[0] += 1
                    out.zero_()
                addr, ctx, pyfn = api._as_fn(f, m, n, DEV, 1)
                api._call(DEV, [pyfn], pkg._lib.lib().fdb_jacobian, p._h, addr, ctx, x.data_ptr(), None, fx.data_ptr(),
                          None, float("nan"), float("nan"), 1.0, None)
                torch.cuda.synchronize()
                calls.append(count[0])
            assert calls[0] == calls[1] == p.info()["fcalls_per_jacobian"], (m, n, fdtype, calls)


def test_mirror_reuse_graph_and_points(pkg, api):
    """finite_difference_jacobian_ on a SparseMatrixCSR: the CSR plan, reused and graph-replayed with x changed in place;
    f sees the points of the COO slot route, in the same order; a dense J with that sparsity takes the COO route."""
    L = pkg._lib
    A = PATTERNS["random_unsorted"]
    m, n = A.shape
    M = pkg.SparseMatrixCSR.from_scipy(A)
    cv = pkg.matrix_colors(M)
    rng = np.random.default_rng(12)
    for fdtype in ("forward", "central"):
        for use_graph in (0, 1):
            x = torch.from_numpy(rng.uniform(-2, 2, n)).to(DEV)
            cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device=DEV), fdtype, colorvec=cv, sparsity=M,
                                      use_graph=use_graph)
            f = _Ell(pkg, A, 2)
            for it in range(3):
                x.copy_(torch.from_numpy(rng.uniform(-2, 2, n)))
                M.nzval.fill_(float("nan"))
                pkg.finite_difference_jacobian_(M, f.fn, x, cache)
                torch.cuda.synchronize()
                assert cache._last_plan.info()["jkind"] == L.FDB_J_CSR
                ref = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
                _jac(pkg, _coo_plan(api, A, cv.cpu().numpy(), fdtype), _Ell(pkg, A, 2), x, ref, fdtype)
                assert_same_bits(M.nzval, ref, f"{fdtype} graph={use_graph} call {it}", allow_nan=False)
    # the points, recorded by a Python f
    small = PATTERNS["tall"]
    Ms = pkg.SparseMatrixCSR.from_scipy(small)
    ns = small.shape[1]
    a, b, d = (torch.from_numpy(np.random.default_rng(s_).uniform(-1, 1, ns)).to(DEV) for s_ in (3, 4, 5))
    for fdtype in ("forward", "central"):
        seen = {}
        for route in ("csr", "coo"):
            pts = []

            def f(fx, xx, pts=pts):
                pts.append(xx.clone())
                y = xx * xx                     # the band's three diagonals, elementwise (a deterministic f)
                fx.zero_()
                fx[:ns] += a * y
                fx[1:ns + 1] += b * y
                fx[:ns - 1] += d[1:] * y[1:]
            x = torch.from_numpy(np.random.default_rng(8).uniform(-2, 2, small.shape[1])).to(DEV)
            J = Ms.similar() if route == "csr" else pkg.zeros_colmajor(*small.shape)
            cache = pkg.JacobianCache(x, torch.zeros(small.shape[0], dtype=torch.float64, device=DEV), fdtype,
                                      colorvec=pkg.matrix_colors(Ms), sparsity=Ms)
            pkg.finite_difference_jacobian_(J, f, x, cache)
            torch.cuda.synchronize()
            seen[route] = (torch.stack(pts).cpu().numpy(), J)
        assert_same_bits(seen["csr"][0], seen["coo"][0], f"{fdtype} points")
        dense = seen["coo"][1].cpu().numpy()
        Md = seen["csr"][1]
        assert_same_bits(Md.nzval.cpu().numpy(), dense[small.tocoo().row, small.tocoo().col], f"{fdtype} dense J")


def _trace(fn):
    """(kernel names, memset count) of fn() under torch.profiler, with the throwaway launches of _util.traced on both
    sides: a session's first and last device records can be missing from its trace in a process that has profiled
    before."""
    import json
    import os
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pad = torch.empty(1, device=DEV)
        for _ in range(64):
            pad.fill_(0.0)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        for _ in range(64):
            pad.fill_(0.0)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            events = json.load(fh)["traceEvents"]
    kernels = [e["name"] for e in events if e.get("cat") == "kernel"]
    memsets = sum(1 for e in events if "memset" in (e.get("cat", "") + e.get("name", "")).lower()
                  and e.get("cat") not in ("cuda_runtime", "cuda_driver"))     # device-side fills only
    return kernels, memsets


def test_profile_shows_csr_kernel_and_no_fill(pkg, api):
    A = PATTERNS["random_unsorted"]
    n = A.shape[1]
    x = torch.from_numpy(np.random.default_rng(1).uniform(-2, 2, n)).to(DEV)
    cv = _valid_coloring(A, np.random.default_rng(1))
    p = _csr_plan(api, A, cv, "forward")
    J = torch.empty(A.nnz, dtype=torch.float64, device=DEV)
    f = _Ell(pkg, A, 1)
    _jac(pkg, p, f, x, J, "forward")
    kernels, memsets = _trace(lambda: _jac(pkg, p, f, x, J, "forward"))
    assert sum("diff_scatter_csr" in k for k in kernels) == 1, kernels
    assert memsets == 0, kernels
    # the COO slot route on the same buffer does zero-fill J: the trace sees its memset
    q = _coo_plan(api, A, cv, "forward")
    _jac(pkg, q, _Ell(pkg, A, 1), x, J, "forward")
    kernels, memsets = _trace(lambda: _jac(pkg, q, _Ell(pkg, A, 1), x, J, "forward"))
    assert any("diff_scatter_dest" in k for k in kernels) and memsets >= 1, kernels


def test_refusals_before_any_f_call(pkg, api):
    L = pkg._lib
    lib = L.lib()
    o = api._opts(0, 0)

    def create(m, n, rp, cv):
        h = C.c_void_p()
        rpa = np.asarray(rp if rp is not None else [], np.int64)
        cva = np.asarray(cv, np.int64)
        st = lib.fdb_plan_create_csr(C.byref(h), m, n, rpa.ctypes.data if rp is not None else None,
                                     cva.ctypes.data if len(cva) else None, None, C.byref(o))
        if st == 0:
            lib.fdb_plan_destroy(h)
        return st

    assert create(2, 2, None, [1]) == L.FDB_ERR_INVALID
    assert create(2, 2, [0, 1, 2], [1, 2]) == L.FDB_ERR_INVALID            # rowptr[1] != 1
    assert create(3, 2, [1, 3, 2, 3], [1, 2]) == L.FDB_ERR_INVALID         # decreasing
    assert create(2, 2, [1, 2, 3], [1, 3]) == L.FDB_ERR_INVALID            # column outside 1..n
    assert create(2, 2, [1, 2, 3], [0, 1]) == L.FDB_ERR_INVALID
    assert create(-1, 2, [1], []) == L.FDB_ERR_INVALID
    assert create(1, 2, [1, (1 << 31) + 1], [1]) == L.FDB_ERR_UNSUPPORTED  # nnz >= 2^31, refused before colval is read
    assert create(2, 2, [1, 2, 3], [2, 1]) == L.FDB_OK
    # peer stores are not built for this plan
    A = PATTERNS["tall"]
    p = _csr_plan(api, A, None, "forward")
    arr = (C.c_void_p * 1)(0)
    assert lib.fdb_plan_set_peers(p._h, 0, arr) == L.FDB_ERR_UNSUPPORTED


def test_colouring_equals_csc_and_is_valid(pkg):
    L = pkg._lib
    lib = L.lib()
    rng = np.random.default_rng(21)
    for t in range(52):
        m, n = int(rng.integers(1, 400)), int(rng.integers(1, 400))
        A = sp.random(m, n, density=float(rng.uniform(0.002, 0.05)), format="csr", random_state=int(rng.integers(1 << 30)))
        A.data[:] = 1.0
        if t % 4 == 0:                                   # unsorted columns within rows
            for i in range(m):
                s, e = A.indptr[i], A.indptr[i + 1]
                A.indices[s:e] = rng.permutation(A.indices[s:e])
        rp, cl = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
        T = A.tocsc()
        T.sort_indices()
        cp, rv = T.indptr.astype(np.int64) + 1, T.indices.astype(np.int64) + 1
        out_r = torch.zeros(n, dtype=torch.int64, device=DEV)
        out_c = torch.zeros(n, dtype=torch.int64, device=DEV)
        nc_r, nc_c, nr = C.c_int64(), C.c_int64(), C.c_int64()
        d_rp, d_cl = torch.from_numpy(rp).to(DEV), torch.from_numpy(cl).to(DEV)
        src = (d_rp.data_ptr(), d_cl.data_ptr()) if t % 2 else (rp.ctypes.data, cl.ctypes.data if A.nnz else None)
        L.check(lib.fdb_matrix_colors_csr(m, n, *src, out_r.data_ptr(), C.byref(nc_r), C.byref(nr)))
        L.check(lib.fdb_matrix_colors_csc(m, n, cp.ctypes.data, rv.ctypes.data if A.nnz else None, out_c.data_ptr(),
                                          C.byref(nc_c), C.byref(nr)))
        torch.cuda.synchronize()
        a, b = out_r.cpu().numpy(), out_c.cpu().numpy()
        assert np.array_equal(a, b) and nc_r.value == nc_c.value, t
        # valid according to scipy: no row holds two columns of one colour
        for i in range(m):
            c = a[A.indices[A.indptr[i]:A.indptr[i + 1]]]
            assert len(set(c.tolist())) == len(c), (t, i)
        k = C.c_int64()
        L.check(lib.fdb_check_coloring_csr(m, n, rp.ctypes.data, cl.ctypes.data if A.nnz else None, a.ctypes.data,
                                           C.byref(k)))
        assert k.value == 0
        bad = np.ones(n, np.int64)
        k2 = C.c_int64()
        L.check(lib.fdb_check_coloring_csr(m, n, rp.ctypes.data, cl.ctypes.data if A.nnz else None, bad.ctypes.data,
                                           C.byref(k2)))
        k3 = C.c_int64()
        L.check(lib.fdb_check_coloring_csc(m, n, cp.ctypes.data, rv.ctypes.data if A.nnz else None, bad.ctypes.data,
                                           C.byref(k3)))
        assert k2.value == k3.value
    M = pkg.SparseMatrixCSR.from_scipy(A)
    assert pkg.check_coloring(M, pkg.matrix_colors(M).cpu().numpy()) == 0


def test_groups_and_shared_j_ranks(pkg, api):
    from finitediff_jl_b200 import distributed
    A = PATTERNS["random_unsorted"]
    m, n = A.shape
    cv = _valid_coloring(A, np.random.default_rng(5))
    cv[::11] = 0
    x = torch.from_numpy(np.random.default_rng(5).uniform(-2, 2, n)).to(DEV)
    for fdtype in ("forward", "central"):
        ref = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
        _jac(pkg, _coo_plan(api, A, cv, fdtype), _Ell(pkg, A, 4), x, ref, fdtype)
        # a [0, 0] group
        M = pkg.SparseMatrixCSR.from_scipy(A)
        M.nzval.fill_(float("nan"))
        g = distributed.GroupJacobian(M, cv, fdtype, [0, 0])
        fs = [_Ell(pkg, A, 4).fn, _Ell(pkg, A, 4).fn]
        g.run(fs, x, torch.zeros(m, dtype=torch.float64, device=DEV))
        torch.cuda.synchronize()
        assert_same_bits(M.nzval, ref, f"{fdtype} group", allow_nan=False)
        # a world = 2 shared_j pair on one buffer, LPT partition
        J = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
        calls = 0
        for r in (0, 1):
            p = _csr_plan(api, A, cv, fdtype, rank=r, world=2, partition=1, shared_j=1)
            f = _Ell(pkg, A, 4)
            _jac(pkg, p, f, x, J, fdtype)
            calls += f.ctx.calls
            owner = np.zeros(int(cv.max()), np.int32)
            pkg._lib.check(pkg._lib.lib().fdb_plan_color_owner(p._h, owner.ctypes.data_as(C.POINTER(C.c_int32)), len(owner)))
        assert_same_bits(J, ref, f"{fdtype} shared_j", allow_nan=False)


class _Tridiag:
    def __init__(self, L, N):
        self.ctx = L.TridiagCtx(N, 0)
        self.addr = C.cast(L.synth().fdbs_tridiag, C.c_void_p).value


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_c2_size_tridiagonal(pkg, api, fdtype):
    """N = 10^7 tridiagonal (3 cyclic colours): the CSR plan against the CSC route's nzval, permuted, and the COO route."""
    L = pkg._lib
    N = 10_000_000
    A = sp.diags([np.ones(N - 1), np.ones(N), np.ones(N - 1)], [-1, 0, 1], format="csr")
    A.sort_indices()
    cv = (np.arange(N) % 3 + 1).astype(np.int64)
    x = torch.empty(N, dtype=torch.float64, device=DEV)
    L.synth().fdbs_fill_x(x.data_ptr(), N, 0x5EED, None)
    out = {}
    for route in ("csr", "coo"):
        fn = _Tridiag(L, N)
        plan = (_csr_plan if route == "csr" else _coo_plan)(api, A, cv, fdtype)
        J = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
        _jac(pkg, plan, fn, x, J, fdtype)
        out[route] = (J, fn.ctx.calls)
        del plan
    assert_same_bits(out["csr"][0], out["coo"][0], f"C2 {fdtype} vs COO", allow_nan=False)
    assert out["csr"][1] == out["coo"][1]
    del out["coo"]
    # the CSC route: tridiagonal CSC slot order is column-major; permute on the device
    T = sp.csr_matrix((np.arange(A.nnz, dtype=np.float64), A.indices, A.indptr), shape=A.shape).tocsc()
    perm = torch.from_numpy(T.data.astype(np.int64)).to(DEV)
    cp, rv = T.indptr.astype(np.int64) + 1, T.indices.astype(np.int64) + 1
    fn = _Tridiag(L, N)
    p = _plan(api, "csc", (N, N, cp.ctypes.data, rv.ctypes.data, L.FDB_J_CSC_NZVAL, None, None, 0, cv.ctypes.data), fdtype,
              (cp, rv, cv))
    Jc = torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=DEV)
    _jac(pkg, p, fn, x, Jc, fdtype)
    viacsc = torch.empty_like(Jc)
    viacsc[perm] = Jc
    assert_same_bits(out["csr"][0], viacsc, f"C2 {fdtype} vs CSC", allow_nan=False)
    assert fn.ctx.calls == out["csr"][1]
