"""The out-of-place Jacobian on the device against the C restatement oop_oracle/ on patterns and colourings that can break
the code depending on the pattern's shape: the zero-dropping compaction oop_compact (column pointers of columns that
start inside a tile, at its first element, at position 1024 or at E, empty and trailing columns, oop_tile_first_col), the
per-entry colour read of the fused compaction at 8, 16 and 32 bits, the dense branch's FULL compaction (`e % m`) and
oop_dense_finish with m != n, the several-groups (kCopy) form with colour-0 columns, batched callbacks and the group form.
tests/test_gpu_oop.py covers the result kinds' semantics on the tridiagonal pattern; this file covers the shapes.

Every comparison is a bit compare (assert_same_bits) of the result kind, size, colptr, rowval and values, with the exact
f call count and the caller's x left unchanged.  Coloured plans feed the restatement the device's step sizes, as
tests/test_gpu_oop.py does.  f is the native ELL rows function fdbs_ellrows (complex step: fdbs_ellrows_c) and the
restatement drives its CPU twin synth_ellrows / synth_ellrows_c (oracle/synth_fns.c); the pattern is the function's
dependence plus spurious structural entries, whose quotients are exactly zero, so the compaction drops entries unevenly
across tiles.  Python callbacks use the same sum on torch tensors (one elementwise kernel per operation, nothing fused)."""
import ctypes as C
import re

import numpy as np
import pytest
import scipy.sparse as sps

from _util import assert_same_bits, fdb_env, traced
from oop_oracle import fd_oop_oracle as OO
from test_gpu_oop import NpF, TorchF, _check_points, _sparse_proto, _to_host_result, assert_same_result

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

_f64p = C.POINTER(C.c_double)


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


# ------------------------------------------------------------------------------------------------ f and its twins
class Ell:
    """f_i = sum_p coef[p,i]*x[cols[p,i]] (left to right) + 0.1*x0^2, x0 = x[cols[0,i]]; ELL layout [K][m]"""

    def __init__(self, cols, coef):
        self.cols = np.ascontiguousarray(cols, dtype=np.int32)
        self.coef = np.ascontiguousarray(coef, dtype=np.float64)
        self.K, self.m = self.cols.shape
        self.dev = {}                          # device copies, made on first use

    def _on(self, device):
        device = torch.device(device)
        if device not in self.dev:
            self.dev[device] = (torch.from_numpy(self.cols).to(device), torch.from_numpy(self.coef).to(device),
                                torch.from_numpy(self.cols.astype(np.int64)).to(device))
        return self.dev[device]

    def native(self, pkg, complex_=False, device="cuda"):
        """the device function as a NativeFn, and its context (ctx.calls counts the points)"""
        d_cols, d_coef, _ = self._on(device)
        ctx = pkg._lib.EllCtx(self.m, self.K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
        fn = pkg._lib.synth().fdbs_ellrows_c if complex_ else pkg._lib.synth().fdbs_ellrows
        return pkg.NativeFn(C.cast(fn, C.c_void_p).value, ctx), ctx

    def torch_f(self, x):
        """the same operations on a (n,) or (batch, n) float64 CUDA tensor"""
        _, coef, cols = self._on(x.device)
        x0 = x[..., cols[0]]
        s = coef[0] * x0
        for p in range(1, self.K):
            s = s + coef[p] * x[..., cols[p]]
        return s + 0.1 * (x0 * x0)


class Twin:
    """synth_ellrows / synth_ellrows_c on numpy arrays, counting (and optionally recording) the points"""

    def __init__(self, ell, oracle, complex_=False, record=True):
        self.ell, self.record, self.complex_ = ell, record, complex_
        self.ctx = oracle.SynthEllCtx(ell.m, ell.K, ell.cols.ctypes.data_as(C.POINTER(C.c_int32)),
                                      ell.coef.ctypes.data_as(_f64p), 1)
        self.fn = oracle.lib().synth_ellrows_c if complex_ else oracle.lib().synth_ellrows
        self.points, self.calls = [], 0

    def __call__(self, x):
        self.calls += 1
        x = np.ascontiguousarray(x)
        if self.record:
            self.points.append(x.copy())
        out = np.zeros(self.ell.m, np.complex128 if self.complex_ else np.float64)
        self.fn(C.byref(self.ctx), out.ctypes.data_as(_f64p), x.ctypes.data_as(_f64p))
        return out


def csc_of(m, n, ell, er=(), ec=()):
    """CSC pattern (1-based Int64) of the function's dependence plus the structural entries (er, ec)"""
    r = np.concatenate([np.tile(np.arange(m), ell.K), np.asarray(er, np.int64)])
    c = np.concatenate([ell.cols.reshape(-1).astype(np.int64), np.asarray(ec, np.int64)])
    A = sps.csc_matrix((np.ones(len(r)), (r, c)), shape=(m, n))
    A.sum_duplicates()
    A.sort_indices()
    return A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1


def greedy_colouring(m, n, cp, rv, rng, skip=()):
    """a valid colouring (no two columns of one colour share a row), columns visited in random order; `skip` columns
    get colour 0"""
    row_used = [set() for _ in range(m)]
    cv = np.zeros(n, np.int64)
    skip = set(skip)
    for c in rng.permutation(n):
        if c in skip:
            continue
        rows = rv[cp[c] - 1:cp[c + 1] - 1] - 1
        bad = set().union(*(row_used[r] for r in rows)) if len(rows) else set()
        k = 1
        while k in bad:
            k += 1
        cv[c] = k
        for r in rows:
            row_used[r].add(k)
    return cv


def is_valid(cp, rv, cv):
    """no row holds two entries of one colour >= 1 (the dense result's _make_Ji condition)"""
    ecol = np.repeat(np.arange(len(cp) - 1), np.diff(cp))
    k = cv[ecol]
    keep = k >= 1
    pairs = (rv[keep] - 1) * (int(cv.max(initial=0)) + 1) + k[keep]
    return np.unique(pairs).size == pairs.size


def spread_ids(cv, C, rng):
    """the colours 1..max(cv) mapped increasingly onto ids in 1..C with C used: most of 1..C become empty colours"""
    used = int(cv.max(initial=0))
    if used < 1:
        return cv
    ids = np.sort(rng.choice(np.arange(1, C), used - 1, replace=False)) if used > 1 else np.zeros(0, np.int64)
    ids = np.concatenate([ids, [C]]).astype(np.int64)
    out = cv.copy()
    out[cv >= 1] = ids[cv[cv >= 1] - 1]
    return out


def make_x(rng, n, nan=False):
    x = rng.uniform(-1.5, 1.5, n)
    x[rng.random(n) < 0.08] = 0.0
    x[rng.random(n) < 0.08] = -0.0
    if nan:
        x[rng.integers(0, n)] = np.nan
    return x


# ------------------------------------------------------------------------------------------------ one coloured case
def run_csc(pkg, oracle, ell, x, cp, rv, cv, *, fd="forward", sparse=True, dir=1.0, steps=(None, None), f_in=False,
            max_batch=1, scratch=0, sm=None, record=True, native_twin=False, band=None, what=""):
    """The device's finite_difference_jacobian(f, x, cache, f_in; sparsity, colorvec[, jac_prototype]) with the native
    ELL function, compared with the restatement; returns (device result, plan).  An invalid colouring with a dense result
    must raise on both sides.  band: a band sparsity object (BandedMatrix, Diagonal, ...) handed to the device instead of
    the CSC (cp, rv), which must then be the CSC of its entry set; the restatement still receives (cp, rv)."""
    m, n = ell.m, len(x)
    complex_ = fd == "complex"
    f, ctx = ell.native(pkg, complex_)
    xd = torch.from_numpy(x.copy()).cuda()
    x_before = xd.clone()
    S = pkg.SparseMatrixCSC(m, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    tk = {"sparsity": S if band is None else band, "colorvec": cv}
    lk = {"sparsity": (m, n, cp, rv), "colorvec": cv}
    if sparse:
        tk["jac_prototype"] = S
        lk["jac_prototype"] = ("sparse", m, n)
    twin = Twin(ell, oracle, complex_, record)
    fin_h = twin(x) if f_in else None
    twin.calls, twin.points = 0, []
    plan_kw = {"max_batch": max_batch}
    if scratch:
        plan_kw["scratch_bytes"] = scratch
    cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd, **plan_kw)
    relstep, absstep = steps
    kw = {} if complex_ else {"relstep": relstep, "absstep": absstep, "dir": dir}
    if not sparse and not is_valid(cp, rv, cv):
        with pytest.raises(pkg._lib.FdbError, match="invalid colouring"):
            pkg.finite_difference_jacobian(f, xd, cache, None, **kw, **tk)
        with pytest.raises(OO.OracleThrows):
            OO.jacobian_oop(twin, x, fd, None, eps_override=[0.0] * int(cv.max()), **lk)
        return None, None
    fin_d = torch.from_numpy(fin_h).cuda() if f_in else None
    with fdb_env(SM_COUNT=sm):
        res = pkg.finite_difference_jacobian(f, xd, cache, fin_d, **kw, **tk)
        torch.cuda.synchronize()
    assert_same_bits(xd, x_before, f"{what}: the caller's x")
    plan = cache._last_plan
    Cn = max(int(cv.max()), 0)
    eps = None if complex_ else list(plan.eps()[:Cn])
    rel = pkg.default_relstep(fd) if relstep is None else relstep
    okw = {} if complex_ else {"relstep": rel, "absstep": absstep, "dir": dir}
    if native_twin:
        fn = oracle.native_fn("synth_ellrows_c" if complex_ else "synth_ellrows")
        want = OO.jacobian_oop((C.cast(fn, C.c_void_p).value, twin.ctx), x, fd, fin_h, eps_override=eps, **okw, **lk)
    else:
        want = OO.jacobian_oop(twin, x, fd, fin_h, eps_override=eps, **okw, **lk)
        assert twin.calls == ctx.calls, f"{what}: {ctx.calls} device calls, the restatement made {twin.calls}"
    calls = 2 * Cn if fd == "central" else Cn + (1 if fd == "forward" and not f_in else 0)
    assert ctx.calls == calls, f"{what}: {ctx.calls} calls, expected {calls}"
    h = _to_host_result(res)
    if sparse:
        assert h[0] == "sparse" and h[1:3] == (m, n), what
        assert h[3].shape == (n + 1,) and h[3][0] == 1 and h[3][-1] == len(h[4]) + 1, f"{what}: colptr ends"
    else:
        assert h[0] == "dense" and h[1].shape == (m, n), what
    assert_same_result(res, want, what)
    return res, plan


# ------------------------------------------------------------------------------------------------ (a) random CSC problems
def random_problem(seed, lo=1, hi=401):
    rng = np.random.default_rng(seed)
    m, n = int(rng.integers(lo, hi)), int(rng.integers(lo, hi))
    K = int(rng.integers(1, 5))
    live = np.flatnonzero(rng.random(n) >= rng.random() * 0.6)     # ragged: a random share of the columns stays empty
    if live.size == 0:
        live = np.array([int(rng.integers(0, n))])
    ell = Ell(rng.choice(live, size=(K, m)), rng.uniform(-1, 1, size=(K, m)))
    extra = int(rng.integers(0, m + 1))
    er = rng.integers(0, m, extra)
    ec = np.where(rng.random(extra) < 0.5, rng.choice(live, extra), rng.integers(0, n, extra))
    cp, rv = csc_of(m, n, ell, er, ec)
    fd = ["forward", "central", "complex"][int(rng.integers(0, 3))]
    sparse = bool(rng.random() < 0.6)
    if not sparse and m * n > 4_000_000:
        sparse = True
    r = rng.random()
    if r < 0.05:
        cv = np.zeros(n, np.int64)                                    # every column at colour 0
    elif r < 0.55 or (not sparse and r < 0.9):
        cv = greedy_colouring(m, n, cp, rv, rng)                      # valid
    else:
        cv = rng.integers(1, int(rng.integers(1, 13)) + 1, n).astype(np.int64)   # most likely invalid
    if rng.random() < 0.3:
        cv[rng.random(n) < 0.15] = 0                                  # columns without a colour
    if rng.random() < 0.3 and cv.max() >= 1:
        cv = spread_ids(cv, int(cv.max()) * int(rng.integers(2, 4)), rng)   # unused colours
    kw = dict(fd=fd, sparse=sparse, max_batch=int(rng.integers(1, 5)))
    if fd != "complex":
        kw["dir"] = [1.0, -1.0, 0.3][int(rng.integers(0, 3))]
        kw["steps"] = [(None, None), (1e-3, 0.0), (0.0, 1e-4), (1e-2, None)][int(rng.integers(0, 4))]
        kw["f_in"] = fd == "forward" and bool(rng.random() < 0.35)
        if rng.random() < 0.3:      # a budget of 1-2 slabs: the outputs come in several groups (the kCopy compaction)
            kw["scratch"] = int(8 * (m + 2) * (2 if fd == "central" else 1) * int(rng.integers(1, 3)) + 64)
    x = make_x(rng, n, nan=bool(rng.random() < 0.15))
    return ell, x, cp, rv, cv, kw


@pytest.mark.parametrize("sm", [None, 1, 3])
@pytest.mark.parametrize("seed", range(150))
def test_random_csc(pkg, oracle, seed, sm):
    ell, x, cp, rv, cv, kw = random_problem(seed)
    what = f"seed={seed} sm={sm} m={ell.m} n={len(x)} E={len(rv)} C={cv.max()} {kw}"
    run_csc(pkg, oracle, ell, x, cp, rv, cv, sm=sm, what=what, **kw)


@pytest.mark.parametrize("sm", [None, 1, 3])
@pytest.mark.parametrize("seed", range(4))
def test_random_csc_mid_size(pkg, oracle, seed, sm):
    """m, n of 10^4-10^5: the compaction takes many tiles per block (sparse results; colourings random, so mostly
    invalid, and with colour 0)"""
    rng = np.random.default_rng(9000 + seed)
    m, n = int(rng.integers(10_000, 100_001)), int(rng.integers(10_000, 100_001))
    K = 3
    live = np.flatnonzero(rng.random(n) >= 0.2)
    ell = Ell(rng.choice(live, size=(K, m)), rng.uniform(-1, 1, size=(K, m)))
    extra = m // 2
    cp, rv = csc_of(m, n, ell, rng.integers(0, m, extra), rng.integers(0, n, extra))
    cv = rng.integers(0, int(rng.integers(4, 25)), n).astype(np.int64)
    cv[0] = max(int(cv.max()), 1)
    fd = ["forward", "central", "complex", "forward"][seed]
    kw = dict(fd=fd, max_batch=[1, 4, 2, 3][seed], scratch=8 * (m + 2) * 2 + 64 if seed == 3 else 0)
    if fd != "complex":
        kw["dir"] = -1.0 if seed % 2 else 1.0
    run_csc(pkg, oracle, ell, make_x(rng, n, nan=seed == 1), cp, rv, cv, sm=sm, record=False,
            what=f"mid seed={seed} sm={sm} m={m} n={n} E={len(rv)}", **kw)


# ------------------------------------------------------------------------------------------------ (b) compaction edges
def edge_problem(m, lens, keep, rng, sink=None):
    """A pattern with the given column lengths (distinct rows per column) and the ELL function whose dependence is
    exactly the entries where `keep` is true (keep: [E] bools in storage order).  Under the valid colouring built here a
    kept entry's quotient is not zero and every other entry's is exactly zero, so the compaction keeps exactly `keep`.
    Rows without a kept entry read the `sink` column, which has colour 0 (it is never perturbed)."""
    n = len(lens)
    cp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + 1
    rv = np.concatenate([np.sort(rng.choice(m, L, replace=False)) for L in lens] or [np.zeros(0, np.int64)])
    rv = rv.astype(np.int64) + 1
    ecol = np.repeat(np.arange(n), lens)
    if sink is None:
        empty = np.flatnonzero(np.asarray(lens) == 0)
        sink = int(empty[0]) if empty.size else 0
    keep = np.asarray(keep, bool) & (ecol != sink)
    per_row = [[] for _ in range(m)]
    for e in np.flatnonzero(keep):
        per_row[rv[e] - 1].append(int(ecol[e]))
    K = max(1, max(len(r) for r in per_row))
    cols = np.full((K, m), sink, np.int64)
    coef = np.zeros((K, m))
    for i, r in enumerate(per_row):
        if r:
            cols[:len(r), i] = r
            cols[len(r):, i] = r[0]                           # padding: coefficient 0
            coef[:len(r), i] = rng.uniform(0.5, 1.5, len(r)) * rng.choice([-1.0, 1.0], len(r))
    cv = greedy_colouring(m, n, cp, rv, rng, skip=[sink])
    return Ell(cols, coef), cp, rv, cv, keep


def _lens_edge(name, rng):
    """(m, column lengths, keep rule) of each deliberately built compaction edge"""
    r = lambda k, a, b: list(rng.integers(a, b, k))
    if name == "leading_empty":
        return 500, [0] * 7 + r(400, 1, 7), 0.7
    if name == "empty_run_at_1024":            # columns 256..264 empty, starting at entry 1024; 530..536 at 2048
        return 600, [4] * 256 + [0] * 9 + [4] * 256 + [0] * 7 + r(100, 1, 5), 0.7
    if name == "trailing_empty_E1024":
        return 400, [4] * 256 + [0] * 6, 0.7
    if name == "trailing_empty_E2048":
        return 400, [4] * 512 + [0] * 3, 0.7
    if name == "trailing_empty_E1029":
        return 400, [4] * 257 + [1] + [0] * 5, 0.7
    if name == "long_column":                  # tiles 1 and 2 lie inside column 50: they start no column
        return 3500, r(50, 1, 5) + [3100] + r(50, 1, 5), 0.7
    if name == "many_starts":                  # about 3000 columns start in the first tile
        return 1500, list((rng.random(3100) < 0.33).astype(int)) + r(200, 1, 5), 0.7
    if name == "dropped_tile":                 # every candidate of tile 1 dropped, tiles 0 and 2 keep entries
        return 700, r(800, 1, 7), "tile1"
    if name == "all_dropped":
        return 600, r(500, 0, 6), 0.0
    raise KeyError(name)


EDGES = ["leading_empty", "empty_run_at_1024", "trailing_empty_E1024", "trailing_empty_E2048", "trailing_empty_E1029",
         "long_column", "many_starts", "dropped_tile", "all_dropped", "arrowhead"]


def build_edge(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "arrowhead":                    # column 0 holds every row, row 0 every column, plus the diagonal
        n = 300
        lens = [n] + [2] * (n - 1)
        cp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + 1
        rv = np.concatenate([np.arange(n)] + [np.array([0, c]) for c in range(1, n)]).astype(np.int64) + 1
        per_row = [list(range(n))] + [[0, i] for i in range(1, n)]
        K = n
        cols = np.array([r + [r[0]] * (K - len(r)) for r in per_row]).T
        coef = np.array([list(rng.uniform(0.5, 1.5, len(r))) + [0.0] * (K - len(r)) for r in per_row]).T
        cv = greedy_colouring(n, n, cp, rv, rng)      # every column its own colour: C = 300, a 16-bit table
        return Ell(cols, coef), cp, rv, cv, np.ones(len(rv), bool), n
    m, lens, rule = _lens_edge(name, rng)
    E = int(np.sum(lens))
    if rule == "tile1":
        keep = (rng.random(E) < 0.6) & ((np.arange(E) < 1024) | (np.arange(E) >= 2048))
    else:
        keep = rng.random(E) < rule
    ell, cp, rv, cv, keep = edge_problem(m, lens, keep, rng)
    return ell, cp, rv, cv, keep, len(lens)


@pytest.mark.parametrize("sm", [None, 1, 3])
@pytest.mark.parametrize("name", EDGES)
def test_compaction_edges(pkg, oracle, name, sm):
    ell, cp, rv, cv, keep, n = build_edge(name)
    rng = np.random.default_rng(len(name))
    x = rng.uniform(0.5, 1.5, n) * rng.choice([-1.0, 1.0], n)
    runs = [dict(fd="forward"), dict(fd="central", dir=-1.0), dict(fd="forward", scratch=8 * (ell.m + 2) + 64)]
    if sm is None:
        runs.append(dict(fd="forward", sparse=False))
    for kw in runs:
        what = f"{name} sm={sm} E={len(rv)} {kw}"
        res, _ = run_csc(pkg, oracle, ell, x, cp, rv, cv, sm=sm, record=False, what=what, **kw)
        if kw.get("sparse", True):
            # the pattern was built so that exactly the `keep` entries survive
            assert res.nnz == int(keep.sum()), what
            kept_pos = np.flatnonzero(keep)
            assert np.array_equal(res.rowval.cpu().numpy(), rv[kept_pos]), what


def test_compaction_edge_shapes():
    """the edges are what their names say (a check of the builder, so that a change to it cannot silently lose one)"""
    _np = np
    for name in EDGES:
        _, cp, rv, cv, keep, n = build_edge(name)
        E = len(rv)
        starts = cp[:-1] - 1
        if name == "empty_run_at_1024":
            assert (starts == 1024).sum() >= 9 and (starts == 2048).sum() >= 7
        if name.startswith("trailing_empty"):
            assert E == int(name[len("trailing_empty_E"):]) and (starts == E).sum() >= 3
        if name == "long_column":
            assert _np.diff(cp).max() > 2048 and not ((starts >= 1024) & (starts < 3072)).any()
        if name == "many_starts":
            assert ((starts >= 0) & (starts < 1024)).sum() > 1024
        if name == "dropped_tile":
            assert not keep[1024:2048].any() and keep[:1024].any() and keep[2048:].any()
        if name == "all_dropped":
            assert E > 0 and not keep.any()
        if name == "leading_empty":
            assert (starts[:7] == 0).all() and cp[7] == 1


# ------------------------------------------------------------------------------------------------ (c) wide colour tables
def _wide_problem(C_):
    rng = np.random.default_rng(C_)
    m, n = 650, 600
    ell = Ell(rng.integers(0, n, size=(3, m)), rng.uniform(-1, 1, size=(3, m)))
    cp, rv = csc_of(m, n, ell, rng.integers(0, m, 100), rng.integers(0, n, 100))
    cv = greedy_colouring(m, n, cp, rv, rng)
    cv[rng.random(n) < 0.1] = 0
    cv = spread_ids(cv, C_, rng)
    return ell, cp, rv, cv, make_x(rng, n)


@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("sparse", [True, False])
def test_wide_colour_table_16bit(pkg, oracle, sparse, fd):
    ell, cp, rv, cv, x = _wide_problem(300)
    res, plan = run_csc(pkg, oracle, ell, x, cp, rv, cv, fd=fd, sparse=sparse, max_batch=4, record=False,
                        what=f"C=300 {fd} sparse={sparse}")
    assert plan.info()["color_bits"] == 16
    if sparse:
        # the fused compaction reads 16-bit entry colours: read its instantiation from a trace of the same call
        f, _ = ell.native(pkg)
        xd = torch.from_numpy(x).cuda()
        S = pkg.SparseMatrixCSC(ell.m, len(x), torch.from_numpy(cp), torch.from_numpy(rv),
                          torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
        cache = pkg.JacobianCache(xd, torch.zeros(ell.m, dtype=torch.float64, device="cuda"), fd, max_batch=4)
        ev = traced(lambda: pkg.finite_difference_jacobian(f, xd, cache, sparsity=S, colorvec=cv, jac_prototype=S))
        mode = "0" if fd == "forward" else "1"
        pat = re.compile(r"oop_compact<\s*(false|\(bool\)0)\s*,\s*(\(int\))?" + mode + r"\s*,\s*unsigned short\s*>")
        names = {k for k, _ in ev if "oop_compact" in k}
        assert any(pat.search(k) for k in names), names


@pytest.mark.parametrize("sparse", [True, False])
def test_wide_colour_table_32bit(pkg, oracle, sparse):
    """C = 70 000: a 32-bit colour table, nearly every colour empty (each still calls f).  The dense result is checked
    against the restatement's sparse result scattered into +0.0 (each structural slot holds 0.0 + q under a valid
    colouring, and a dropped entry is +-0.0): the restatement's dense form takes O(C m n)."""
    ell, cp, rv, cv, x = _wide_problem(70_000)
    assert cv.max() == 70_000
    if sparse:
        _, plan = run_csc(pkg, oracle, ell, x, cp, rv, cv, max_batch=4, record=False, native_twin=True, what="C=70000")
        assert plan.info()["color_bits"] == 32
        return
    m, n = ell.m, len(x)
    f, ctx = ell.native(pkg)
    xd = torch.from_numpy(x).cuda()
    S = pkg.SparseMatrixCSC(m, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), "forward", max_batch=4)
    J = pkg.finite_difference_jacobian(f, xd, cache, sparsity=S, colorvec=cv)
    plan = cache._last_plan
    assert plan.info()["color_bits"] == 32 and ctx.calls == 70_001
    fn = oracle.native_fn("synth_ellrows")
    twin = Twin(ell, oracle)
    want = OO.jacobian_oop((C.cast(fn, C.c_void_p).value, twin.ctx), x, "forward", sparsity=(m, n, cp, rv), colorvec=cv,
                           jac_prototype=("sparse", m, n), eps_override=list(plan.eps()[:70_000]))
    ref = np.zeros((m, n))
    cols = np.repeat(np.arange(n), np.diff(want[3]))
    ref[want[4] - 1, cols] = 0.0 + want[5]
    assert_same_bits(J, ref, "C=70000 dense")


# ------------------------------------------------------------------------------------------------ (d) the dense branch, m != n
def gathers(rng, m, n):
    """f_i = (a_i * x[p1_i]) * x[p2_i] + b_i * x[p3_i]: single IEEE operations on torch (1-D or batched) or numpy"""
    p1, p2, p3 = (rng.integers(0, n, m) for _ in range(3))
    a, b = rng.uniform(-2, 2, m), rng.uniform(-2, 2, m)
    dev = {}

    def f(x, lib=torch):
        if lib is np:
            return (a * x[p1]) * x[p2] + b * x[p3]
        if x.device not in dev:
            dev[x.device] = [torch.from_numpy(t).to(x.device) for t in (p1, p2, p3, a, b)]
        q1, q2, q3, ta, tb = dev[x.device]
        return (ta * x[..., q1]) * x[..., q2] + tb * x[..., q3]
    return f


DENSE_SHAPES = [(1023, 9), (1024, 17), (1025, 8), (2047, 12), (2048, 5), (2049, 6), (3072, 30), (5, 40), (1, 33),
                (30_000, 8)]


@pytest.mark.parametrize("kind", ["raw", "dense_proto", "sparse_proto"])
@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("m,n", DENSE_SHAPES)
def test_dense_branch_m_ne_n(pkg, m, n, fd, kind):
    rng = np.random.default_rng(m * 7 + n)
    fn = gathers(rng, m, n)
    x = make_x(rng, n)
    C_ = int(rng.integers(max(1, n // 2), n + 1)) if n > 1 else 1
    cv = rng.integers(1, C_ + 1, n).astype(np.int64)
    cv[int(rng.integers(0, n))] = C_
    extra = int(rng.integers(0, 3))
    tk, lk = {"colorvec": cv}, {"colorvec": cv}
    if kind == "dense_proto":
        tk["jac_prototype"] = torch.zeros((C_ + extra, m), dtype=torch.float64, device="cuda").t()
        lk["jac_prototype"] = ("dense", m, C_ + extra)
    elif kind == "sparse_proto":
        tk["jac_prototype"] = _sparse_proto(pkg, m, C_ + extra)
        lk["jac_prototype"] = ("sparse", m, C_ + extra)
    for sm in ([None, 1] if m == 30_000 else [None]):
        xd = torch.from_numpy(x).cuda()
        x_before = xd.clone()
        tf, nf = TorchF(fn, record=m <= 4096), NpF(fn)
        dir = -1.0 if fd == "forward" else 0.3
        with fdb_env(SM_COUNT=sm):
            cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd)
            res = pkg.finite_difference_jacobian(tf, xd, cache, dir=dir, **tk)
            torch.cuda.synchronize()
        what = f"{kind} {fd} m={m} n={n} C={C_} sm={sm}"
        assert_same_bits(xd, x_before, f"{what}: the caller's x")
        want = OO.jacobian_oop(nf, x, fd, relstep=pkg.default_relstep(fd), dir=dir, m=m, **lk)
        h = _to_host_result(res)
        ncols = C_ if kind == "raw" else C_ + extra
        assert (h[1].shape if h[0] == "dense" else h[1:3]) == (m, ncols), what
        assert_same_result(res, want, what)
        calls = (1 + C_) if fd == "forward" else 2 * C_
        assert len(nf.points) == calls, what
        if tf.record:
            _check_points(tf, nf, what)


# ------------------------------------------------------------------------------------------------ (e) batched callbacks
class BatchedF:
    """A batched out-of-place f (f.batched = True): records every invocation as the list of points it received"""
    batched = True

    def __init__(self, fn):
        self.fn, self.calls = fn, []

    def __call__(self, x):
        h = x.detach().cpu().numpy()
        self.calls.append([h.copy()] if x.dim() == 1 else [r.copy() for r in h])
        return self.fn(x)


def _split_central(seq, want_pts, start, max_b, what):
    """Check that `seq` (the points f saw after position `start` of the restatement's sequence) is the restatement's
    central sequence (x+e_k, x-e_k per colour) regrouped in blocks: the plus points of up to max_b consecutive colours,
    then their minus points.  Returns the block sizes."""
    pts = want_pts[start:]
    C_ = len(pts) // 2
    assert len(seq) == 2 * C_, f"{what}: {len(seq)} points, expected {2 * C_}"
    k, i, blocks = 0, 0, []
    while k < C_:
        b = 0
        while k + b < C_ and i + b < len(seq) and np.array_equal(seq[i + b].view(np.uint64), pts[2 * (k + b)].view(np.uint64)):
            b += 1
        # an all-equal plus / minus pair (a zero step) is matched as plus: shrink b until the minus block fits
        while b > 0 and not all(np.array_equal(seq[i + b + j].view(np.uint64), pts[2 * (k + j) + 1].view(np.uint64))
                                for j in range(b)):
            b -= 1
        assert 1 <= b <= max_b, f"{what}: point {i} starts no block of plus points then minus points (colour {k + 1})"
        blocks.append(b)
        i += 2 * b
        k += b
    return blocks


def _batched_problem(pkg, kind, seed):
    rng = np.random.default_rng(seed)
    if kind in ("raw", "dense_proto", "sparse_proto"):
        m, n = 13, 10
        ell = Ell(rng.integers(0, n, size=(2, m)), rng.uniform(-1, 1, size=(2, m)))
        C_ = 9
        cv = rng.integers(1, C_ + 1, n).astype(np.int64)
        cv[0] = C_
        tk, lk = {"colorvec": cv}, {"colorvec": cv}
        if kind == "dense_proto":
            tk["jac_prototype"] = torch.zeros((C_ + 1, m), dtype=torch.float64, device="cuda").t()
            lk["jac_prototype"] = ("dense", m, C_ + 1)
        elif kind == "sparse_proto":
            tk["jac_prototype"] = _sparse_proto(pkg, m, C_ + 1)
            lk["jac_prototype"] = ("sparse", m, C_ + 1)
        return ell, make_x(rng, n), tk, lk, C_
    m, n = 50, 40
    ell = Ell(rng.integers(0, n, size=(2, m)), rng.uniform(-1, 1, size=(2, m)))
    cp, rv = csc_of(m, n, ell, rng.integers(0, m, 20), rng.integers(0, n, 20))
    cv = greedy_colouring(m, n, cp, rv, rng)
    cv[3] = 0
    S = pkg.SparseMatrixCSC(m, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    tk, lk = {"sparsity": S, "colorvec": cv}, {"sparsity": (m, n, cp, rv), "colorvec": cv}
    if kind == "csc_sparse":
        tk["jac_prototype"] = S
        lk["jac_prototype"] = ("sparse", m, n)
    return ell, make_x(rng, n), tk, lk, int(cv.max())


ALL_KINDS = ["raw", "dense_proto", "sparse_proto", "csc_dense", "csc_sparse"]


@pytest.mark.parametrize("fd", ["forward", "central"])
@pytest.mark.parametrize("kind", ALL_KINDS)
@pytest.mark.parametrize("form", ["batched", "per_point", "native"])
def test_batched_callbacks(pkg, oracle, form, kind, fd):
    """max_batch = 3 on the cache.  A batched Python f receives (batch, n) points; a Python f without `batched` is called
    once per point of each batch; a NativeFn receives the batch.  Values bit for bit; every point in order: forward
    f(x) then the colours ascending, central the plus points of a batch of colours then their minus points"""
    ell, x, tk, lk, C_ = _batched_problem(pkg, kind, 40 + ALL_KINDS.index(kind))
    m, n = ell.m, len(x)
    xd = torch.from_numpy(x).cuda()
    x_before = xd.clone()
    cache = pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd, max_batch=3)
    if form == "batched":
        f = BatchedF(ell.torch_f)
    elif form == "per_point":
        f = TorchF(ell.torch_f)
    else:
        f, ctx = ell.native(pkg)
    res = pkg.finite_difference_jacobian(f, xd, cache, **tk)
    torch.cuda.synchronize()
    what = f"{form} {kind} {fd}"
    assert_same_bits(xd, x_before, f"{what}: the caller's x")
    twin = Twin(ell, oracle)
    eps = list(cache._last_plan.eps()[:C_]) if "sparsity" in lk else None
    want = OO.jacobian_oop(twin, x, fd, relstep=pkg.default_relstep(fd), eps_override=eps, m=m, **lk)
    assert_same_result(res, want, what)
    calls = 1 + C_ if fd == "forward" else 2 * C_
    assert twin.calls == calls, what
    if form == "native":
        assert ctx.calls == calls, what
        return
    if form == "batched":
        sizes = [len(c) for c in f.calls]
        seq = [p for c in f.calls for p in c]
        assert max(sizes) <= 3 and (C_ < 2 or max(sizes) > 1), f"{what}: invocation sizes {sizes}"
    else:
        seq = f.points
    # forward: the mirror's f(x) (one 1-D call), then the colours ascending in the reference's order
    start = 0
    if fd == "forward":
        assert len(seq) == len(twin.points), f"{what}: {len(seq)} points, expected {len(twin.points)}"
        for i, (a, b) in enumerate(zip(seq, twin.points)):
            assert_same_bits(a, b, f"{what}: point {i}")
        if form == "batched":
            assert sizes[0] == 1 and f.calls[0][0].ndim == 1
        return
    blocks = _split_central(seq, twin.points, start, 3, what)
    if form == "batched":
        assert sizes == [b for b in blocks for _ in (0, 1)], f"{what}: invocations {sizes} for blocks {blocks}"


# ------------------------------------------------------------------------------------------------ (f) groups
def device_sets():
    sets = [[0, 0], [0, 0, 0], [0, 0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets.append([0, 1])
    return sets


@pytest.mark.parametrize("devs", device_sets())
@pytest.mark.parametrize("seed", range(6))
def test_group_random(pkg, oracle, fdist, devs, seed):
    """random CSC problems from the generator above (forward / central) through GroupJacobianOOP, round-robin and LPT,
    against the restatement and the one-device result; seed 5 is a C = 300 dense result (the members' own slots decoded
    from a 16-bit colour table)"""
    if seed == 5:
        ell, cp, rv, cv, x = _wide_problem(300)
        kw = {"fd": "central", "sparse": False, "dir": -1.0}     # spurious entries: -0.0 quotients, +0.0 in the result
    else:
        s = 500 + seed * 37
        ell, x, cp, rv, cv, kw = random_problem(s)
        while kw["fd"] == "complex":                 # groups run forward / central plans
            s += 1
            ell, x, cp, rv, cv, kw = random_problem(s)
        if not kw["sparse"] and not is_valid(cp, rv, cv):
            cv = greedy_colouring(ell.m, len(x), cp, rv, np.random.default_rng(seed))
        if seed % 2 == 0:
            cv[:: 7] = 0
    m, n = ell.m, len(x)
    fd, sparse = kw["fd"], kw["sparse"]
    partition = seed % 2
    what = f"group {devs} seed={seed} {fd} sparse={sparse} partition={partition} C={cv.max()}"
    single, plan = run_csc(pkg, oracle, ell, x, cp, rv, cv, fd=fd, sparse=sparse, dir=kw.get("dir", 1.0),
                           steps=kw.get("steps", (None, None)), record=False, what=what)
    xd = torch.from_numpy(x).cuda(devs[0])
    x_before = xd.clone()
    S = pkg.SparseMatrixCSC(m, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device=xd.device))
    with torch.cuda.device(devs[0]):
        g = fdist.GroupJacobianOOP(devs, fd, colorvec=cv, sparsity=S, jac_prototype=S if sparse else None,
                                   partition=partition)
        members = [ell.native(pkg, device=f"cuda:{d}") for d in devs]
        res = g.run([f for f, _ in members], xd, relstep=kw.get("steps", (None, None))[0],
                    absstep=kw.get("steps", (None, None))[1], dir=kw.get("dir", 1.0))
        torch.cuda.synchronize()
    assert_same_bits(xd, x_before, f"{what}: the caller's x")
    assert_same_result(res, _to_host_result(single), f"{what}: against one device")
    Cn = int(cv.max())
    calls = sum(ctx.calls for _, ctx in members)
    assert calls == (2 * Cn if fd == "central" else Cn + 1), f"{what}: {calls} calls"
    twin = Twin(ell, oracle, record=False)
    rel = pkg.default_relstep(fd) if kw.get("steps", (None, None))[0] is None else kw["steps"][0]
    want = OO.jacobian_oop(twin, x, fd, relstep=rel, absstep=kw.get("steps", (None, None))[1], dir=kw.get("dir", 1.0),
                           eps_override=list(plan.eps()[:Cn]), sparsity=(m, n, cp, rv), colorvec=cv,
                           jac_prototype=("sparse", m, n) if sparse else None)
    assert_same_result(res, want, f"{what}: against the restatement")
    g.close()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_rank_slots_with_a_16bit_colour_table(pkg, world):
    """C = 300, a dense result of a CSC sparsity, one rank plan at a time on J prefilled with -0.0: a rank's `+ 0.0` runs
    over exactly the slots of the colours it owns (decoded from the 16-bit entry colours), so every other slot stays -0.0
    and its own slots hold the one-device values"""
    ell, cp, rv, cv, x = _wide_problem(300)
    m, n = ell.m, len(x)
    L = pkg._lib
    xd = torch.from_numpy(x).cuda()
    col = np.repeat(np.arange(n), np.diff(cp))

    def rank_run(rank, w):
        o = pkg.api._opts(L.FDB_FORWARD, 0, rank=rank, world=w, shared_j=w > 1)
        h = C.c_void_p()
        L.check(L.lib().fdb_oop_plan_create_csc(C.byref(h), m, n, cp.ctypes.data, rv.ctypes.data, cv.ctypes.data,
                                                L.FDB_OOP_DENSE, m, C.byref(o)))
        plan = pkg.Plan(h.value)
        f, _ = ell.native(pkg)
        J = torch.full((n, m), -0.0, dtype=torch.float64, device="cuda").t()
        out = L.OopOut()
        out.J = J.data_ptr()
        L.check(L.lib().fdb_jacobian_oop(plan.handle, C.c_void_p(f.address), f.ctx_ptr, xd.data_ptr(), C.byref(out), None,
                                         None, L.STEP_DEFAULT, L.STEP_DEFAULT, -1.0,
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        return plan, J.cpu().numpy()

    one, ref = rank_run(0, 1)
    assert one.info()["color_bits"] == 16
    union = np.zeros((m, n), bool)
    for r in range(world):
        plan, got = rank_run(r, world)
        owner = plan.color_owner()[:300]
        mine = (cv[col] >= 1) & (owner[np.maximum(cv[col], 1) - 1] == r)
        own = np.zeros((m, n), bool)
        own[rv[mine] - 1, col[mine]] = True
        assert_same_bits(got[own], ref[own], f"rank {r}/{world}: its own slots")
        assert (np.signbit(got[~own]) & (got[~own] == 0)).all(), f"rank {r}/{world} wrote a slot it does not own"
        union |= own
    struct = np.zeros((m, n), bool)
    struct[rv - 1, col] = True
    assert np.array_equal(union, struct & (cv[None, :] >= 1))


def test_several_groups_colourless_columns(pkg, oracle):
    """The sparse result with its f outputs in several groups reads candidates the in-place scatter wrote; the entries of
    columns without a colour are defined only by the scatter's zero for them.  The plan's candidate buffer is allocated
    over freed device memory that held NaN, so a candidate nobody writes would show up as a kept NaN."""
    rng = np.random.default_rng(77)
    m, n = 20_000, 18_000
    ell = Ell(rng.integers(0, n, size=(3, m)), rng.uniform(-1, 1, size=(3, m)))
    cp, rv = csc_of(m, n, ell, rng.integers(0, m, 5000), rng.integers(0, n, 5000))
    cv = rng.integers(1, 6, n).astype(np.int64)
    cv[rng.random(n) < 0.25] = 0
    x = make_x(rng, n)
    for fd in ("forward", "central"):
        junk = torch.full((1 << 27,), float("nan"), dtype=torch.float64, device="cuda")      # 1 GiB
        del junk
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        _, plan = run_csc(pkg, oracle, ell, x, cp, rv, cv, fd=fd, scratch=8 * (m + 2) * (2 if fd == "central" else 1) + 64,
                          record=False, what=f"several groups, colour 0, {fd}")
        assert plan.info()["n_groups"] > 1


# ------------------------------------------------------------------------------------------------ (g) maximum(colorvec) < 1
@pytest.mark.parametrize("cacheless", [False, True])
@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
@pytest.mark.parametrize("proto", ["raw", "dense", "sparse"])
@pytest.mark.parametrize("colour", [0, -3])
def test_dense_branch_without_colours(pkg, colour, proto, fd, cacheless):
    """sparsity = nothing and maximum(colorvec) < 1: the reference's colour loop is empty and it returns
    zero(jac_prototype) (jacobians.jl:307-309, 333) after f(x) in forward mode; without a prototype it throws"""
    m, n = 7, 5
    idx = torch.tensor([0, 1, 2, 3, 4, 0, 2], device="cuda")
    pts = []

    def f(v):
        pts.append(v.detach().cpu().numpy().copy())
        return (v * v)[idx]
    x = np.array([0.5, -0.0, 1.25, -2.0, 0.0])
    xd = torch.from_numpy(x).cuda()
    x_before = xd.clone()
    cv = np.full(n, colour, np.int64)
    kw = {"colorvec": cv}
    if proto == "dense":
        kw["jac_prototype"] = torch.full((n + 1, m), -0.0, dtype=torch.float64, device="cuda").t()
    elif proto == "sparse":
        kw["jac_prototype"] = _sparse_proto(pkg, m, n + 1)
    cache = None if cacheless else pkg.JacobianCache(xd, torch.zeros(m, dtype=torch.float64, device="cuda"), fd)
    call = lambda: pkg.finite_difference_jacobian(f, xd, fd if cacheless else cache, **kw)
    if proto == "raw":
        with pytest.raises(pkg._lib.FdbError, match="no column"):
            call()
        return
    res = call()
    torch.cuda.synchronize()
    assert_same_bits(xd, x_before, "the caller's x")
    h = _to_host_result(res)
    if proto == "dense":
        assert h[0] == "dense" and h[1].shape == (m, n + 1)
        assert_same_bits(h[1], np.zeros((m, n + 1)), "zero(jac_prototype): +0.0 everywhere")
    else:
        assert h[0] == "sparse" and h[1:3] == (m, n + 1)
        assert np.array_equal(h[3], np.ones(n + 2, np.int64)) and h[4].size == 0 and h[5].size == 0
    assert len(pts) == (1 if (fd == "forward" or cacheless) else 0), len(pts)
    for p in pts:
        assert_same_bits(p.real if np.iscomplexobj(p) else p, x, "f(x)")
    # the restatement agrees
    lk = {"colorvec": cv, "jac_prototype": (proto, m, n + 1)}
    want = OO.jacobian_oop(lambda v: (v * v)[idx.cpu().numpy()], x, fd, m=m, cacheless=cacheless, **lk)
    assert_same_result(res, want, f"{proto} {fd} cacheless={cacheless}")


@pytest.mark.parametrize("proto", ["dense", "sparse"])
def test_group_dense_branch_without_colours(pkg, fdist, proto):
    """the group form with maximum(colorvec) < 1: every rank > 0 is idle, the root alone forms zero(jac_prototype)"""
    m, n = 6, 4
    x = torch.tensor([0.5, -0.0, 1.5, 2.0], dtype=torch.float64, device="cuda")
    cv = np.zeros(n, np.int64)
    proto_t = (torch.full((n + 2, m), -0.0, dtype=torch.float64, device="cuda").t() if proto == "dense"
               else _sparse_proto(pkg, m, n + 2))
    for fd in ("forward", "central"):
        g = fdist.GroupJacobianOOP([0, 0, 0], fd, colorvec=cv, jac_prototype=proto_t)
        fs = [TorchF(lambda v: torch.cat([v, v[:2]])) for _ in range(3)]
        res = g.run(fs, x)
        torch.cuda.synchronize()
        h = _to_host_result(res)
        if proto == "dense":
            assert_same_bits(h[1], np.zeros((m, n + 2)), f"group {fd}")
        else:
            assert h[1:3] == (m, n + 2) and np.array_equal(h[3], np.ones(n + 3, np.int64)) and h[4].size == 0
        assert [len(f.points) for f in fs] == ([1, 0, 0] if fd == "forward" else [0, 0, 0])
        g.close()
