"""Multi-wave parity: every hot-path kernel with several tiles (grid-stride steps) per block, bit for bit.

The kernels walk their data in 1024-element tiles with a grid-stride loop whose grid is sized from the SM count, so at the
sizes a test can afford on a 132-SM H100 most blocks see one tile: the second and later iterations of a tile loop, the TMA
pipeline refill of the staged scatter and its mbarrier parity flip, the reverse walk over several tiles and the choice of
the block that takes the partial last tile would run only at full size.  FDB_SM_COUNT=k makes a plan size its grids as if
the device had k SMs (launch geometry only), which reaches the same loops with problems a hundred times smaller.

Every case holds the parity bar of the other GPU tests: J bit-identical to the oracle fed the device step sizes, the
device step sizes within rtol 1e-13 of the oracle's own, the f! call count exact, and the path the plan took read from
plan.info().  The kernels a call ran are read from a torch.profiler trace: their grids prove the tile counts per block,
and the template arguments in the demangled names prove which staged-scatter instantiation an A/B switch reached."""
import ctypes as C
import json
import os
import re
import tempfile

import numpy as np
import pytest
import scipy.sparse as sps

from _util import assert_same_bits, band_csc, fdb_env, tridiag_csc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TILE = 1024
THREADS = 256
FD = {"forward": 0, "central": 1}
REACHED = {}     # kernel -> largest tiles (grid-stride steps) per block seen in this module


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REACHED:
        print("\nlargest tiles (grid-stride steps) per block:")
        for k in sorted(REACHED):
            print(f"  {k:28s} {REACHED[k]:8.1f}")


# ------------------------------------------------------------------------------------------------ profiler trace
def traced(fn):
    """Run fn() under torch.profiler (CUDA activity); return [(kernel name, grid x, grid y, shared memory bytes)]."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # kernel records at either end of a session can be missing from its trace: the first few once the profiler has
        # sat idle for a minute or so in a process, the last one when the session stops right after it (seen for the
        # staged scatter, the last launch of a forward call).  Throwaway launches take those places on both sides.
        pad = torch.empty(1, device="cuda")
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
    out = []
    for e in sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0)):
        a = e.get("args", {})
        g = a.get("grid", [1, 1, 1])
        out.append((e["name"], int(g[0]), int(g[1]), int(a.get("shared memory", -1))))
    return out


def launches(kernels, name):
    return [k for k in kernels if re.search(r"\b" + name + r"<|\b" + name + r"\(", k[0])]


def note(kernels, name, units, need=None):
    """Launches of kernel `name`: units of work per launch (a number, or a list in launch order) over the grid's x size.
    Records the largest quotient and asserts it reaches `need`."""
    ks = launches(kernels, name)
    assert ks, f"{name} did not run: {[k[0][:60] for k in kernels]}"
    per = [units] * len(ks) if np.isscalar(units) else list(units)
    assert len(per) == len(ks), (name, len(per), len(ks))
    best = max(u / k[1] for u, k in zip(per, ks))
    REACHED[name] = max(REACHED.get(name, 0.0), best)
    if need is not None:
        assert best >= need, f"{name}: {best:.2f} tiles per block < {need} (grids {[k[1] for k in ks]})"
    return best


def _targs(name):
    """Template arguments of a demangled kernel name, split at the top-level commas."""
    s = name[name.index("<") + 1: name.rindex(">(")]
    out, depth, cur = [], 0, ""
    for ch in s:
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    out.append(cur.strip())
    return out


def staged_instance(kernels):
    """(MINB, PREFETCH, PACKED, EMPTYBAR, BAND) of the one diff_scatter_staged launch, and its shared memory."""
    ks = launches(kernels, "diff_scatter_staged")
    assert len(ks) == 1, [k[0] for k in kernels]
    a = _targs(ks[0][0])[-5:]
    b = lambda v: v in ("true", "1", "(bool)1")
    return (int(a[0]), b(a[1]), b(a[2]), b(a[3]), b(a[4])), ks[0][3]


# ------------------------------------------------------------------------------------------------ pattern families
def _csc(m, n, r, c):
    A = sps.csc_matrix((np.ones(len(r)), (r, c)), shape=(m, n))
    A.sum_duplicates()
    A.sort_indices()
    return A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1


def band_with_holes(m, n, l, u, seed):
    """A clipped band with about 10 % of its entries removed and extra entries just below it in every 20th column:
    row-local, but not an exact band."""
    rng = np.random.default_rng(seed)
    colptr, rowval = band_csc(m, n, l, u)
    c = np.repeat(np.arange(n), np.diff(colptr))
    r = rowval - 1
    keep = rng.random(len(r)) >= 0.1
    xc = np.arange(0, n, 20)
    xr = xc + u + 1 + rng.integers(0, 3, len(xc))
    ok = xr < m
    return _csc(m, n, np.concatenate([r[keep], xr[ok]]), np.concatenate([c[keep], xc[ok]]))


def stencil(g, points):
    """5- or 9-point stencil on a g x g grid (neighbours outside the grid dropped)."""
    idx = np.arange(g * g)
    i, j = idx % g, idx // g
    offs = [(0, 0), (-1, 0), (1, 0), (0, -1), (0, 1)]
    if points == 9:
        offs += [(-1, -1), (1, -1), (-1, 1), (1, 1)]
    rr, cc = [], []
    for di, dj in offs:
        ii, jj = i + di, j + dj
        ok = (ii >= 0) & (ii < g) & (jj >= 0) & (jj < g)
        rr.append(idx[ok])
        cc.append((ii + jj * g)[ok])
    return _csc(g * g, g * g, np.concatenate(rr), np.concatenate(cc))


def block_tridiag(nb, b):
    """Block-tridiagonal pattern: nb x nb blocks of b x b, blocks (I, J) with |I - J| <= 1 full."""
    n = nb * b
    c = np.arange(n)
    B = c // b
    lo, hi = np.maximum(B - 1, 0) * b, np.minimum(B + 2, nb) * b
    cnt = hi - lo
    cols = np.repeat(c, cnt)
    rows = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt) + np.repeat(lo, cnt)
    return _csc(n, n, rows, cols)


def indexed_patterns():
    """name -> (m, n, colptr, rowval): row-local CSC patterns that are not exact bands (the indexed staged form).
    Sizes: >= 3 full tiles per block at k = 1 (at most 8 resident blocks), staging windows inside the 46 KB cap."""
    out = {}
    for name, (m, n, l, u) in {"holes": (40000, 36000, 3, 1), "holes_wide": (30000, 34000, 1, 5)}.items():
        out[name] = (m, n) + band_with_holes(m, n, l, u, seed=len(name))
    out["lap5"] = (100 * 100, 100 * 100) + stencil(100, 5)
    out["lap9"] = (70 * 70, 70 * 70) + stencil(70, 9)
    out["blocktri"] = (3000 * 4, 3000 * 4) + block_tridiag(3000, 4)
    return out


_PATTERNS = {}


def pattern(name):
    if name not in _PATTERNS:
        _PATTERNS.update(indexed_patterns())
    return _PATTERNS[name]


def colouring(kind, n, C, seed=0):
    rng = np.random.default_rng(seed + 17 * C)
    if kind == "cyclic":
        return (np.arange(n) % C + 1).astype(np.int64)
    if kind == "random":                       # arbitrary, structurally invalid colouring; every colour used
        cv = rng.integers(1, C + 1, n).astype(np.int64)
        cv[:C] = np.arange(1, C + 1)
        return cv
    cv = (np.arange(n) % C + 1).astype(np.int64)   # "zero": some columns without a valid colour
    cv[rng.integers(0, n, max(1, n // 50))] = 0
    cv[:C] = np.arange(1, C + 1)
    return cv


# ------------------------------------------------------------------------------------------------ harness
class Problem:
    """A CSC problem with an ELL f! (row i depends on K entries of its own pattern row), run on the GPU and the oracle."""

    def __init__(self, pkg, oracle, m, n, colptr, rowval, cv, fdtype, *, K=3, seed=1):
        self.pkg, self.oracle = pkg, oracle
        self.m, self.n, self.colptr, self.rowval, self.cv, self.fdtype = m, n, colptr, rowval, cv, fdtype
        self.E = len(rowval)
        rng = np.random.default_rng(seed)
        # f! dependence inside the pattern: row r reads K random entries of pattern row r (rows without entries read x[r])
        A = sps.csc_matrix((np.ones(self.E), (rowval - 1, np.repeat(np.arange(n), np.diff(colptr)))), shape=(m, n)).tocsr()
        cnt = np.diff(A.indptr)
        pick = A.indptr[:-1, None] + (rng.random((m, K)) * np.maximum(cnt, 1)[:, None]).astype(np.int64)
        cols = np.where(cnt[:, None] > 0, A.indices[np.minimum(pick, max(A.nnz - 1, 0))], np.minimum(np.arange(m), n - 1)[:, None])
        self.colsT = np.ascontiguousarray(cols.T.astype(np.int32))
        self.coefT = np.ascontiguousarray(rng.uniform(-1, 1, size=(K, m)))
        self.K = K
        self.xh = rng.uniform(-2, 2, n)      # |x| <= 2: sums of squares far from fp64 overflow / underflow
        self._own = {}

    def octx(self):
        return self.oracle.SynthEllCtx(self.m, self.K, self.colsT.ctypes.data_as(C.POINTER(C.c_int32)),
                                       self.coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)

    def own_eps(self, dirv=1.0, no_drift=False):
        key = (dirv, no_drift)
        if key not in self._own:
            P = self.oracle.Problem.csc_same(self.m, self.n, self.colptr, self.rowval)
            self._own[key] = self.oracle.jacobian(P, np.zeros(self.E), self.oracle.native_fn("synth_ellrows"), self.xh.copy(),
                                                  fdtype=FD[self.fdtype], colorvec=self.cv, dir=dirv, no_drift=no_drift,
                                                  ctx=self.octx())["eps"]
        return self._own[key]

    def run(self, sm_count=None, env=None, *, f_in=False, dirv=1.0, no_drift=False, x_offset=0, j_offset=0,
            dense_J=False, oracle_check=True, profile=False, **opts):
        pkg, dev, L = self.pkg, torch.device("cuda:0"), self.pkg._lib
        m, n, E = self.m, self.n, self.E
        d_cols, d_coef = torch.from_numpy(self.colsT).to(dev), torch.from_numpy(self.coefT).to(dev)
        ctx = L.EllCtx(m, self.K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
        f = pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx, max_batch=opts.get("max_batch", 1))
        xbuf = torch.zeros(n + x_offset, dtype=torch.float64, device=dev)
        x = xbuf[x_offset:]
        x.copy_(torch.from_numpy(self.xh))
        if dense_J:
            J = pkg.zeros_colmajor(m, n, dev)
            J.fill_(float("nan"))
            sp = pkg.SparseMatrixCSC(m, n, torch.from_numpy(self.colptr), torch.from_numpy(self.rowval), None)
        else:
            nzbuf = torch.full((E + j_offset,), float("nan"), dtype=torch.float64, device=dev)
            sp = J = pkg.SparseMatrixCSC(m, n, torch.from_numpy(self.colptr), torch.from_numpy(self.rowval), nzbuf[j_offset:])
        fin_t, kw = None, {}
        if f_in:
            fin = np.zeros(m)
            self.oracle.lib().synth_ellrows(C.byref(self.octx()), fin.ctypes.data_as(C.POINTER(C.c_double)),
                                            self.xh.ctypes.data_as(C.POINTER(C.c_double)))
            fin_t = torch.from_numpy(fin).to(dev)
            kw["f_in"] = fin
        fx = torch.zeros(m, dtype=torch.float64, device=dev)
        cache = pkg.JacobianCache(x.clone(), fx, fx.clone(), self.fdtype, colorvec=self.cv, sparsity=sp, no_drift=no_drift,
                                  **opts)
        call = lambda: pkg.finite_difference_jacobian_(J, f, x, cache, fin_t, dir=dirv)
        with fdb_env(SM_COUNT=sm_count, **(env or {})):
            kernels = traced(call) if profile else (call(), torch.cuda.synchronize(), [])[2]
        plan = cache._last_plan
        eps = plan.eps()
        got = J.cpu().numpy().reshape(-1, order="F") if dense_J else sp.nzval.cpu().numpy()
        res = dict(J=got, eps=eps, info=plan.info(), kernels=kernels, calls=ctx.calls)
        if oracle_check:
            if dense_J:
                P = self.oracle.Problem.csc_to_dense(m, n, self.colptr, self.rowval)
                ref = np.full(m * n, np.nan)
            else:
                P = self.oracle.Problem.csc_same(m, n, self.colptr, self.rowval)
                ref = np.full(E, np.nan)
            r = self.oracle.jacobian(P, ref, self.oracle.native_fn("synth_ellrows"), self.xh.copy(), fdtype=FD[self.fdtype],
                                     colorvec=self.cv, eps_override=eps, no_drift=no_drift, dir=dirv, ctx=self.octx(), **kw)
            assert ctx.calls == r["fcalls"]
            assert_same_bits(got, ref, f"J differs from the oracle at sm_count={sm_count} env={env}")
            np.testing.assert_allclose(eps, self.own_eps(dirv, no_drift), rtol=1e-13)
        return res


def plan_shape(info):
    """plan.info() without device_bytes: the step-size pass keeps one partial row per block, so its buffer follows the grid."""
    return {k: v for k, v in info.items() if k != "device_bytes"}


def staged_bytes(p, info, packed):
    """moved_bytes_scatter of the indexed staged form (fdb_plan_info)."""
    C_ = info["n_colors"]
    nwin = 2 * C_ if p.fdtype == "central" else C_ + 1
    return p.E * (2 + (0 if packed else info["color_bits"] // 8) + 8) + 8 * p.m * nwin


def staged_units(p):
    return p.E // TILE


# ------------------------------------------------------------------------------------------------ A. indexed staged form
INDEXED = [  # (pattern, fdtype, C, colouring)
    ("holes", "forward", 1, "cyclic"), ("holes", "forward", 2, "random"), ("holes", "forward", 3, "zero"),
    ("holes_wide", "forward", 4, "cyclic"), ("holes_wide", "forward", 5, "random"),
    ("blocktri", "forward", 6, "zero"), ("blocktri", "forward", 7, "cyclic"),
    ("lap5", "forward", 5, "cyclic"), ("lap9", "forward", 7, "random"),
    ("holes", "central", 1, "random"), ("holes", "central", 2, "cyclic"), ("holes_wide", "central", 3, "zero"),
    ("blocktri", "central", 4, "random"), ("lap5", "central", 3, "zero"), ("lap9", "central", 4, "cyclic"),
]


@pytest.mark.parametrize("name,fdtype,C_,kind", INDEXED)
def test_indexed_staged_multiwave(pkg, oracle, name, fdtype, C_, kind):
    m, n, colptr, rowval = pattern(name)
    p = Problem(pkg, oracle, m, n, colptr, rowval, colouring(kind, n, C_), fdtype)
    base = p.run()
    for k in (1, 3):
        r = p.run(k, profile=True)
        info = r["info"]
        assert info["staged"] == 1 and info["strategy"] == 0 and info["n_groups"] == 1
        assert info["moved_bytes_scatter"] == staged_bytes(p, info, packed=True)       # indexed, packed: not the band form
        assert plan_shape(info) == plan_shape(base["info"])
        inst, _ = staged_instance(r["kernels"])
        assert inst == (6, False, True, False, False)
        note(r["kernels"], "diff_scatter_staged", staged_units(p), need=3 if k == 1 else None)
        np.testing.assert_allclose(r["eps"], base["eps"], rtol=1e-13)


@pytest.mark.parametrize("sm_count", [1, 3])
def test_indexed_staged_options(pkg, oracle, sm_count):
    # f_in, dir = -1, no_drift and an 8-byte aligned J (the scalar store path), on a pattern whose entry count is a
    # multiple of 1024 (no partial last tile) and on one with a partial last tile
    m, n, colptr, rowval = pattern("holes")
    E1 = (len(rowval) // TILE) * TILE
    cut = np.searchsorted(colptr - 1, E1, side="right") - 1          # whole columns up to an entry count % 1024 == 0
    colptr_a = np.minimum(colptr, colptr[cut])
    for cp, rv in ((colptr, rowval), (colptr_a, rowval[: colptr[cut] - 1])):
        for fdtype in ("forward", "central"):
            p = Problem(pkg, oracle, m, n, cp, rv, colouring("zero", n, 3 if fdtype == "forward" else 2), fdtype, seed=5)
            if fdtype == "forward":
                p.run(sm_count, f_in=True)
                p.run(sm_count, dirv=-1.0)
            r = p.run(sm_count, no_drift=True)
            assert r["info"]["staged"] == 1
            r = p.run(sm_count, j_offset=1, profile=True)
            note(r["kernels"], "diff_scatter_staged", staged_units(p), need=3 if sm_count == 1 else None)
        assert cp is colptr or len(rv) % TILE == 0


# A/B switches: each combination with the staged-scatter instantiation it must reach.  (form, switches, expected
# (MINB, PREFETCH, PACKED, EMPTYBAR, BAND)); a variant letter the dispatch ignores in a form is not listed for it.
SWITCHES = [
    ("packed", {}, (6, False, True, False, False)),
    ("packed", {"STAGED_VARIANT": "6e"}, (6, False, True, True, False)),
    ("stream", {"NO_PACK": 1}, (6, False, False, False, False)),
    ("stream", {"NO_PACK": 1, "STAGED_VARIANT": "6n"}, (6, False, False, False, False)),
    ("stream", {"NO_PACK": 1, "STAGED_VARIANT": "8n"}, (8, False, False, False, False)),
    ("stream", {"NO_PACK": 1, "STAGED_VARIANT": "6p"}, (6, True, False, False, False)),
    ("band", {}, (6, False, False, False, True)),
    ("band", {"STAGED_VARIANT": "8n"}, (8, False, False, False, True)),
    ("band", {"STAGED_VARIANT": "6e"}, (6, False, False, True, True)),
]
for _form in ("packed", "stream", "band"):
    _base = {"NO_PACK": 1} if _form == "stream" else {}
    _inst = next(s[2] for s in SWITCHES if s[0] == _form)
    SWITCHES.append((_form, dict(_base, STAGES=3), _inst))
    SWITCHES += [(_form, dict(_base, REVERSE=v), _inst) for v in range(4)]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_staged_switches_bit_identical(pkg, oracle, fdtype, sm_count):
    C_ = 3 if fdtype == "forward" else 2
    probs = {}
    m, n, colptr, rowval = pattern("holes")
    probs["packed"] = probs["stream"] = Problem(pkg, oracle, m, n, colptr, rowval, colouring("random", n, C_), fdtype, seed=3)
    m = n = 30000
    colptr, rowval = band_csc(m, n, 2, 1)
    probs["band"] = Problem(pkg, oracle, m, n, colptr, rowval, colouring("cyclic", n, C_), fdtype, seed=4)
    base = {form: p.run(sm_count, profile=True) for form, p in probs.items() if form != "stream"}
    smem_default = {}
    for form, env, want in SWITCHES:
        p = probs[form]
        r = p.run(sm_count, env, profile=True, oracle_check=False)
        ref = base["band" if form == "band" else "packed"]
        assert_same_bits(r["eps"], ref["eps"], (form, env), allow_nan=False)
        assert_same_bits(r["J"], ref["J"], (form, env))
        assert r["calls"] == ref["calls"]
        inst, smem = staged_instance(r["kernels"])
        assert inst == want, (form, env, inst)
        if env.get("STAGES") == 3:
            assert smem > smem_default[form] * 1.4, (form, smem, smem_default[form])   # three stages really in flight
        elif len(env) <= 1 or form == "stream":
            smem_default.setdefault(form, smem)
        info = r["info"]
        if form == "band":
            assert info["moved_bytes_scatter"] == 8 * p.E + 8 * p.m * (2 * C_ if fdtype == "central" else C_ + 1)
        else:
            assert info["moved_bytes_scatter"] == staged_bytes(p, info, packed=form == "packed")
        note(r["kernels"], "diff_scatter_staged", staged_units(p), need=3 if sm_count == 1 else None)


# ------------------------------------------------------------------------------------------------ C. the other kernels
@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("no_drift", [False, True])
@pytest.mark.parametrize("max_batch", [1, 4])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_perturb_multiwave(pkg, oracle, fdtype, no_drift, max_batch, sm_count):
    # five colours: one pass builds four points (NP = 4), the next one (NP = 1); tridiagonal -> band-form staged scatter
    m = n = 600_002
    colptr, rowval = tridiag_csc(n)
    p = Problem(pkg, oracle, m, n, colptr, rowval, colouring("random", n, 5), fdtype, seed=6)
    r = p.run(sm_count, no_drift=no_drift, max_batch=max_batch, profile=True)
    nps = {int(_targs(k[0])[-1]) for k in launches(r["kernels"], "perturb_colors")}
    assert nps == {1, 4}
    note(r["kernels"], "perturb_colors", -(-n // TILE), need=3 if sm_count == 1 else None)
    if not no_drift and max_batch == 1:
        r0 = p.run(sm_count, {"REVERSE": 0}, oracle_check=False)      # forward walk: same bits
        assert_same_bits(r0["eps"], r["eps"], allow_nan=False)
        assert_same_bits(r0["J"], r["J"], allow_nan=False)


@pytest.mark.parametrize("C_,kind", [(3, "cyclic"), (7, "random")])
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_eps_depth_bit_identical(pkg, oracle, C_, kind, aligned, sm_count):
    # color_sumsq_reg: DEPTH 2 (two tiles of loads in flight) and DEPTH 1 sum in the same order.  n: 56 full tiles, i.e.
    # 7 per block at k = 1 (three DEPTH-2 steps and one odd tile); x = buf[1:] takes the scalar remainder path throughout
    n = 56 * TILE + 38
    colptr, rowval = tridiag_csc(n)
    p = Problem(pkg, oracle, n, n, colptr, rowval, colouring(kind, n, C_), "forward", seed=7)
    off = 0 if aligned else 1
    r2 = p.run(sm_count, x_offset=off, profile=True)
    r1 = p.run(sm_count, {"EPS_DEPTH": 1}, x_offset=off, profile=True)
    assert_same_bits(r1["eps"], r2["eps"], allow_nan=False)
    assert_same_bits(r1["J"], r2["J"], allow_nan=False)
    d2 = [int(_targs(k[0])[-1]) for k in launches(r2["kernels"], "color_sumsq_reg")]
    d1 = [int(_targs(k[0])[-1]) for k in launches(r1["kernels"], "color_sumsq_reg")]
    assert d2 == [2] and d1 == [1]
    units = n // TILE if aligned else -(-n // TILE)
    note(r2["kernels"], "color_sumsq_reg", units, need=3 if sm_count == 1 else None)
    if aligned:
        g = launches(r2["kernels"], "color_sumsq_reg")[0][1]
        per_block = [len(range(b, units, g)) for b in range(g)]
        assert any(t >= 3 and t % 2 == 1 for t in per_block) or sm_count != 1, per_block   # DEPTH-2 steps + an odd tile


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_list_eps_independent_of_grid(pkg, oracle, fdtype):
    # more than 8 colours on a CSC plan: the step sizes come from the per-colour column lists and depend only on x and
    # the colour's column set — bit-identical whatever the grid.  40 colours do not stage: the gather form
    # (diff_scatter_ident, FULL) scatters.
    n = 100_002
    colptr, rowval = tridiag_csc(n)
    p = Problem(pkg, oracle, n, n, colptr, rowval, colouring("random", n, 40), fdtype, seed=8)
    runs = {k: p.run(k, profile=True, max_batch=4) for k in (None, 1, 3)}
    for k in (1, 3):
        assert_same_bits(runs[k]["eps"], runs[None]["eps"], allow_nan=False)
        assert_same_bits(runs[k]["J"], runs[None]["J"], allow_nan=False)
        assert plan_shape(runs[k]["info"]) == plan_shape(runs[None]["info"])
    assert runs[1]["info"]["staged"] == 0
    note(runs[1]["kernels"], "finalize_eps_lists", 40 / 8)
    note(runs[1]["kernels"], "diff_scatter_ident", -(-p.E // TILE), need=3)
    assert "true" in launches(runs[1]["kernels"], "diff_scatter_ident")[0][0]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_ident_non_full_multiwave(pkg, oracle, fdtype, sm_count):
    # a scratch budget of two slabs: several groups, the storage-order pass with ownership tests (diff_scatter_ident
    # non-FULL) once per group
    n = 60_000
    colptr, rowval = tridiag_csc(n)
    p = Problem(pkg, oracle, n, n, colptr, rowval, colouring("zero", n, 7), fdtype, seed=9)
    small = 8 * (n + 2) * (4 if fdtype == "central" else 2) + 64
    r = p.run(sm_count, scratch_bytes=small, strategy=1, profile=True)
    assert r["info"]["n_groups"] > 1 and r["info"]["strategy"] == 0 and r["info"]["staged"] == 0
    ks = launches(r["kernels"], "diff_scatter_ident")
    assert len(ks) == r["info"]["n_groups"] and all("false" in k[0] for k in ks)
    note(r["kernels"], "diff_scatter_ident", -(-p.E // TILE), need=3 if sm_count == 1 else None)


def random_problem(pkg, oracle, m, n, fdtype, C_, seed):
    """The random-pattern generator of test_gpu_random_parity at mid size: ragged columns, extra structural entries."""
    rng = np.random.default_rng(seed)
    K = 4
    dep = rng.integers(0, n, size=(m, K))
    extra = m
    er, ec = rng.integers(0, m, extra), rng.integers(0, n, extra)
    colptr, rowval = _csc(m, n, np.concatenate([np.repeat(np.arange(m), K), er]), np.concatenate([dep.reshape(-1), ec]))
    cv = rng.integers(0, C_ + 1, n).astype(np.int64)          # about 1 in C+1 columns without a valid colour
    cv[:C_] = np.arange(1, C_ + 1)
    p = Problem(pkg, oracle, m, n, colptr, rowval, cv, fdtype, K=K, seed=seed)
    return p


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("strategy", [2, 3])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_colour_major_multiwave(pkg, oracle, fdtype, strategy, sm_count):
    # colour-major lists: per group of resident colours (f(x) pre-gathered into list order) or in one launch; rank 0
    # zeroes the entries of columns without a valid colour
    m, n, C_ = 50_000, 40_000, 8
    p = random_problem(pkg, oracle, m, n, fdtype, C_, seed=10 + strategy)
    kw = dict(strategy=strategy)
    if strategy == 2:
        kw["scratch_bytes"] = 8 * (m + 2) * (4 if fdtype == "central" else 2) + 64
    r = p.run(sm_count, profile=True, **kw)
    info = r["info"]
    assert info["strategy"] == 1 and info["lists_resident"] == (1 if strategy == 3 else 0)
    col_of = np.repeat(np.arange(n), np.diff(p.colptr))
    per_colour = np.bincount(p.cv[col_of], minlength=C_ + 1)          # [0] = entries of colour-0 columns
    G = info["slabs"]
    seg = [int(per_colour[1 + g:1 + min(g + G, C_)].sum()) for g in range(0, C_, G)] if strategy == 2 else [int(per_colour[1:].sum())]
    need = 3 if sm_count == 1 else None
    note(r["kernels"], "diff_scatter_cm", [-(-s // TILE) for s in seg], need=need)
    note(r["kernels"], "zero_slots", -(-int(per_colour[0]) // THREADS), need=need)
    if strategy == 2 and fdtype == "forward":
        assert info["n_groups"] > 1
        note(r["kernels"], "gather_fx_cm", -(-int(per_colour[1:].sum()) // TILE), need=need)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_dest_scatter_multiwave(pkg, oracle, fdtype, sm_count):
    # CSC sparsity into a dense J: explicit destinations (diff_scatter_dest)
    m = n = 4000
    p = random_problem(pkg, oracle, m, n, fdtype, 6, seed=12)
    r = p.run(sm_count, dense_J=True, profile=True)
    note(r["kernels"], "diff_scatter_dest", -(-p.E // THREADS), need=3 if sm_count == 1 else None)


# ---- banded and dense plans
def banded_run(pkg, oracle, m, n, l, u, C_, fdtype, sm_count, dense=False):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(13)
    x = torch.from_numpy(rng.uniform(-2, 2, n)).to(dev)
    xh = x.cpu().numpy().copy()
    cv = (np.arange(n) % C_ + 1).astype(np.int64)
    cv[rng.integers(0, n, max(1, n // 100))] = 0
    L = pkg._lib
    K = 3
    # f! row r reads K columns inside its band [r - l, r + u] (clipped)
    cols = np.clip(np.arange(m)[:, None] + rng.integers(-l, u + 1, size=(m, K)), 0, n - 1).astype(np.int32)
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(rng.uniform(-1, 1, size=(K, m)))
    d_cols, d_coef = torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev)
    ctx = L.EllCtx(m, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx)
    octx = oracle.SynthEllCtx(m, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    Jb = pkg.BandedMatrix(m, n, l, u, device=dev)
    J = pkg.zeros_colmajor(m, n, dev) if dense else Jb
    (J if dense else Jb.data).fill_(float("nan"))
    fx = torch.zeros(m, dtype=torch.float64, device=dev)
    cache = pkg.JacobianCache(x, fx, fx.clone(), fdtype, colorvec=cv, sparsity=Jb)
    with fdb_env(SM_COUNT=sm_count):
        kernels = traced(lambda: pkg.finite_difference_jacobian_(J, f, x, cache))
    eps = cache._last_plan.eps()
    P = oracle.Problem.banded_to_dense(m, n, l, u) if dense else oracle.Problem.banded(m, n, l, u)
    ref = np.zeros(m * n) if dense else np.full((l + u + 1) * n, np.nan)
    r = oracle.jacobian(P, ref, oracle.native_fn("synth_ellrows"), xh.copy(), fdtype=FD[fdtype], colorvec=cv, eps_override=eps,
                        ctx=octx)
    own = oracle.jacobian(P, np.zeros_like(ref), oracle.native_fn("synth_ellrows"), xh.copy(), fdtype=FD[fdtype], colorvec=cv,
                          ctx=octx)
    got = J.cpu().numpy().reshape(-1, order="F") if dense else Jb.data.cpu().numpy()
    assert ctx.calls == r["fcalls"]
    assert_same_bits(got, ref)
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-13)
    return kernels


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_banded_multiwave(pkg, oracle, fdtype, sm_count):
    need = 3 if sm_count == 1 else None
    for (m, n, l, u) in ((100_000, 100_000, 1, 1), (90_000, 100_000, 3, 1)):           # w = 3, 5: diff_scatter_band
        w = l + u + 1
        ks = banded_run(pkg, oracle, m, n, l, u, w, fdtype, sm_count)
        note(ks, "diff_scatter_band", -(-n // (4096 // w)), need=need)
    # w = 65 >= 2C: quotients pre-divided in place (diff_slabs), then the flat copy into the band storage
    m, n, l, u = 30_000, 32_000, 40, 24
    ks = banded_run(pkg, oracle, m, n, l, u, 5, fdtype, sm_count)
    note(ks, "diff_slabs", -(-m // THREADS), need=need)
    nchunks = -(-(l + u + 1) * n // 64)
    note(ks, "diff_scatter_band_flat", nchunks / 8, need=need)
    # the same band into a dense J: one warp per column (diff_scatter_band_wide)
    m, n = 3000, 3200
    ks = banded_run(pkg, oracle, m, n, l, u, 5, fdtype, sm_count, dense=True)
    note(ks, "diff_scatter_band_wide", n / 8, need=need)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("batch", [1, 7])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_dense_columns_multiwave(pkg, oracle, fdtype, batch, sm_count):
    # sparsity === nothing: replicate_x over n components (grid from the SM count), set_components, diff_columns over
    # m = 1537 rows (odd: the last row takes the scalar path; 768 row pairs = 3 steps of one 256-thread block)
    dev = torch.device("cuda:0")
    m, n = 1537, 6200
    rng = np.random.default_rng(14)
    K = 3
    cols = rng.integers(0, n, size=(m, K)).astype(np.int32)
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(rng.uniform(-1, 1, size=(K, m)))
    d_cols, d_coef = torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev)
    L = pkg._lib
    ctx = L.EllCtx(m, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_ellrows, C.c_void_p).value, ctx, max_batch=batch)
    x = torch.from_numpy(rng.uniform(-2, 2, n)).to(dev)
    J = pkg.zeros_colmajor(m, n, dev)
    J.fill_(float("nan"))
    cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device=dev), fdtype, max_batch=batch)
    with fdb_env(SM_COUNT=sm_count):
        ks = traced(lambda: pkg.finite_difference_jacobian_(J, f, x, cache))
    octx = oracle.SynthEllCtx(m, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    ref = np.zeros(m * n)
    r = oracle.jacobian(oracle.Problem.dense(m, n), ref, oracle.native_fn("synth_ellrows"), x.cpu().numpy().copy(),
                        fdtype=FD[fdtype], ctx=octx)
    assert ctx.calls == r["fcalls"] == (n + 1 if fdtype == "forward" else 2 * n)
    assert_same_bits(cache._last_plan.eps(), r["eps"], allow_nan=False)
    assert_same_bits(J.cpu().numpy().reshape(-1, order="F"), ref, allow_nan=False)
    need = 3 if sm_count == 1 else None
    note(ks, "replicate_x", -(-n // THREADS), need=need)
    assert launches(ks, "set_components")
    note([k for k in ks if "diff_columns" in k[0]][:1], "diff_columns", (m // 2) / THREADS, need=3)


# ------------------------------------------------------------------------------------------------ the switch itself
def test_switch_bites(pkg, oracle):
    # k = 1: the staged scatter, the perturbation pass and the step-size pass run with at least 3x fewer blocks than tiles
    m = n = 600_002
    colptr, rowval = tridiag_csc(n)
    p = Problem(pkg, oracle, m, n, colptr, rowval, colouring("random", n, 3), "forward", seed=15)
    r = p.run(1, {"NO_BAND": 1}, profile=True)
    d = p.run(None, {"NO_BAND": 1}, profile=True)
    assert r["info"]["staged"] == 1
    for name, units in (("diff_scatter_staged", p.E // TILE), ("perturb_colors", -(-n // TILE)),
                        ("color_sumsq_reg", n // TILE)):
        ks, kd = launches(r["kernels"], name), launches(d["kernels"], name)
        assert ks and all(units >= 3 * k[1] for k in ks), (name, units, [k[1] for k in ks])
        assert all(k[1] > ks[0][1] for k in kd), (name, "the default grid must be larger")
        note(r["kernels"], name, units, need=3)


def test_switch_leaves_plan_info_unchanged(pkg, oracle):
    # launch geometry only: no plan decision (strategy, staged, band form, packing, slabs, lists) reads the SM count
    cases = [("holes", "forward", 3), ("lap5", "central", 3)]
    for name, fdtype, C_ in cases:
        m, n, colptr, rowval = pattern(name)
        p = Problem(pkg, oracle, m, n, colptr, rowval, colouring("cyclic", n, C_), fdtype)
        infos = [plan_shape(p.run(k, oracle_check=False)["info"]) for k in (None, 1, 3, 0, 100000, "x")]
        assert all(i == infos[0] for i in infos[1:])
    p = random_problem(pkg, oracle, 20_000, 20_000, "forward", 20, seed=16)
    infos = [plan_shape(p.run(k, oracle_check=False, scratch_bytes=8 * 20_002 * 3)["info"]) for k in (None, 1, 3)]
    assert all(i == infos[0] for i in infos[1:])


def test_out_of_range_row_rejected_multiwave(pkg):
    # plan-time validation on a pattern of about 10^6 entries under k = 1: the bad row index in the last column is found
    n = 333_334
    colptr, rowval = tridiag_csc(n)
    bad = rowval.copy()
    bad[-1] = n + 3
    J = pkg.SparseMatrixCSC(n, n, torch.from_numpy(colptr), torch.from_numpy(rowval), None)
    Jbad = pkg.SparseMatrixCSC(n, n, torch.from_numpy(colptr), torch.from_numpy(bad), None)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    dev = torch.device("cuda:0")
    with fdb_env(SM_COUNT=1):
        pkg.make_plan(J, J, cv, "forward", n, dev)          # the valid pattern plans
        with pytest.raises(pkg._lib.FdbError) as ei:
            pkg.make_plan(Jbad, Jbad, cv, "forward", n, dev)
    assert ei.value.status == pkg._lib.FDB_ERR_INVALID
    assert len(rowval) > 999_000
