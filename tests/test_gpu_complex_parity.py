"""Complex-step colour loop (jacobians.jl:623-648) bit for bit against the oracle, on every J kind and every scatter
kernel the complex path reaches.

The step size is eps(Float64) for every colour, with no norm and no reduction, so every case is compared with the
oracle's own run: no eps_override and no tolerance.  Each case checks
  - J bit for bit (pre-filled with NaN wherever the call has to define every slot),
  - the f! call count (one complex evaluation per colour, no f(x) call),
  - plan.eps() == eps(Float64) for every colour,
  - the caller's x, unchanged bit for bit,
and reads from a torch.profiler trace which kernel instantiation ran, so that a routing change cannot quietly leave a
complex kernel untested.  The synthetic f! is the complex twin of the ELL rows function (fdbs_ellrows_c /
synth_ellrows_c): J depends on each row's coefficients, and the square term makes one entry per row depend on x."""
import ctypes as C
import json
import os
import re
import tempfile

import numpy as np
import pytest
import scipy.sparse as sps

from _util import assert_same_bits, ell_c_numpy, fdb_env, tridiagonal_coo

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps
NAN = float("nan")
REACHED = {}     # complex kernel instantiation -> first test whose trace asserted it


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REACHED:
        print("\ncomplex kernel instantiations and the first test that reached them:")
        for k in sorted(REACHED):
            print(f"  {k:70s} {REACHED[k]}")


# ------------------------------------------------------------------------------------------------ profiler trace
def traced(fn):
    """Run fn() under torch.profiler (CUDA activity); return [(kernel name, grid x)] in launch order."""
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
        out.append((e["name"], int(e.get("args", {}).get("grid", [1, 1, 1])[0])))
    return out


def targs(name):
    """Template arguments of a demangled kernel name, split at the top-level commas ([] for a plain function)."""
    if "<" not in name or ">(" not in name:
        return []
    s = name[name.index("<") + 1: name.rindex(">(")]
    out, depth, cur = [], 0, ""
    for ch in s:
        depth += (ch == "<") - (ch == ">")
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    out.append(cur.strip())
    return out


def launched(kernels, name):
    """[(template arguments, grid x)] of every launch of kernel `name`."""
    pat = re.compile(r"\b" + name + r"[<(]")
    return [(targs(k), g) for k, g in kernels if pat.search(k)]


# the scatter kernels and the position of their MODE template argument (kComplex == 2)
MODE_AT = {"diff_scatter_band_flat": 1, "diff_scatter_band_wide": 1, "diff_scatter_band": 1, "diff_scatter_dest": 1,
           "diff_scatter_ident": 1, "diff_scatter_cm": 0, "diff_columns": 0}


def expect(kernels, name, **args):
    """Assert that `name` ran with the complex-step instantiation (MODE == kComplex, and any other template argument
    given by position without the namespace, e.g. a2=FALSE or a0="CyclicColors"); return those launches.  Records the
    instantiation for the module report."""
    hits = [(t, g) for t, g in launched(kernels, name)
            if (name not in MODE_AT or t[MODE_AT[name]] == "2")
            and all(t[int(k[1:])].replace("fdb::", "") in (v if isinstance(v, tuple) else (v,)) for k, v in args.items())]
    assert hits, f"{name} {args} did not run: {sorted({k[:90] for k, _ in kernels})}"
    key = f"{name}<{', '.join(hits[0][0])}>" if hits[0][0] else name
    REACHED.setdefault(key, os.environ.get("PYTEST_CURRENT_TEST", "?").split(" ")[0])
    return hits


def only_complex_scatters(kernels, desc=""):
    """No forward / central / pre-divided (kCopy) scatter instantiation may run in a complex-step call."""
    for name, at in MODE_AT.items():
        for t, _ in launched(kernels, name):
            assert t[at] == "2", f"{desc}: {name}<{', '.join(t)}> ran in a complex-step call"


TRUE, FALSE = ("true", "1", "(bool)1"), ("false", "0", "(bool)0")


# ------------------------------------------------------------------------------------------------ the synthetic f!
class Ell:
    """An ELL rows function, ELL layout [K][m], on the device (fdbs_ellrows_c) and for the oracle (synth_ellrows_c)."""

    def __init__(self, dev, cols, coef):
        self.cols = np.ascontiguousarray(cols, dtype=np.int32)
        self.coef = np.ascontiguousarray(coef, dtype=np.float64)
        self.K, self.m = self.cols.shape
        self.d_cols, self.d_coef = torch.from_numpy(self.cols).to(dev), torch.from_numpy(self.coef).to(dev)

    def native(self, pkg, max_batch=1):
        ctx = pkg._lib.EllCtx(self.m, self.K, self.d_cols.data_ptr(), self.d_coef.data_ptr(), 0)
        return pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_ellrows_c, C.c_void_p).value, ctx, max_batch=max_batch), ctx

    def octx(self, oracle):
        return oracle.SynthEllCtx(self.m, self.K, self.cols.ctypes.data_as(C.POINTER(C.c_int32)),
                                  self.coef.ctypes.data_as(C.POINTER(C.c_double)), 1)


def random_ell(dev, rng, m, n, K):
    return Ell(dev, rng.integers(0, n, size=(K, m)), rng.uniform(-1, 1, size=(K, m)))


def band_ell(dev, rng, m, n, l, u, K):
    """Row i reads columns inside the band only: max(0, i-l) .. min(n-1, i+u)."""
    i = np.arange(m)
    lo, hi = np.maximum(i - l, 0), np.minimum(i + u, n - 1)
    assert (lo <= hi).all(), "every row must meet the band"
    cols = lo + np.floor(rng.random((K, m)) * (hi - lo + 1)).astype(np.int64)
    return Ell(dev, cols, rng.uniform(-1, 1, size=(K, m)))


def csc_of(m, n, ell, rng, extra=0):
    """CSC pattern (1-based Int64) of the function's dependence plus `extra` spurious structural entries."""
    r = np.concatenate([np.tile(np.arange(m), ell.K), rng.integers(0, m, extra)])
    c = np.concatenate([ell.cols.reshape(-1), rng.integers(0, n, extra)])
    A = sps.csc_matrix((np.ones(len(r)), (r, c)), shape=(m, n))
    A.sum_duplicates()
    A.sort_indices()
    return A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1


def make_x(rng, n):
    x = rng.uniform(-2, 2, n)
    x[rng.random(n) < 0.05] = 0.0
    x[rng.random(n) < 0.05] = -0.0          # the complex point's real part is x + 0.0 (+0.0 for a -0.0)
    return x


def colouring(kind, n, C, rng):
    if kind == "cyclic":
        return (np.arange(n) % C + 1).astype(np.int64)
    cv = rng.integers(1, C + 1, n).astype(np.int64) if kind == "table" else (np.arange(n) % C + 1).astype(np.int64)
    if kind == "zero":                       # columns without a valid colour
        cv[rng.random(n) < 0.1] = 0
    cv[rng.integers(0, n)] = C
    return cv


def dev_x(dev, xh, offset=False):
    if not offset:
        return torch.from_numpy(xh.copy()).to(dev)
    buf = torch.empty(len(xh) + 1, dtype=torch.float64, device=dev)
    x = buf[1:]                              # 8-byte aligned only
    x.copy_(torch.from_numpy(xh))
    return x


def J_csc(pkg, m, n, colptr, rowval, dev, offset=False):
    nnz = len(rowval)
    nz = torch.full((nnz + offset,), NAN, dtype=torch.float64, device=dev)[int(offset):]
    return pkg.SparseMatrixCSC(m, n, torch.from_numpy(colptr), torch.from_numpy(rowval), nz)


def J_dense(pkg, m, n, dev, ld=None, fill=NAN):
    """Column-major (m, n) J with leading dimension ld; returns (J, the flat column-major storage)."""
    ld = m if ld is None else ld
    store = torch.full((n, ld), fill, dtype=torch.float64, device=dev)
    return store.t()[:m, :], store.reshape(-1)


def run(pkg, oracle, dev, J, vals, P, ell, xh, *, cv=None, sparsity=None, plan_kw=None, env=None, x_offset=False,
        trace=True, desc=""):
    """One complex Jacobian through the Python mirror, compared with the oracle's jacobian_complex on the same problem.
    vals: J's flat value storage on the device, laid out as the oracle Problem P stores J.  Returns the kernel trace and
    the plan."""
    plan_kw = dict(plan_kw or {})
    x = dev_x(dev, xh, x_offset)
    f, ctx = ell.native(pkg, plan_kw.get("max_batch", 1))
    fx = torch.zeros(P.m, dtype=torch.float64, device=dev)
    cache = pkg.JacobianCache(x, fx, "complex", colorvec=cv, sparsity=sparsity, **plan_kw)
    ref = vals.cpu().numpy().copy()          # slots the call does not define keep what J held before
    with fdb_env(**(env or {})):
        if trace:
            kernels = traced(lambda: pkg.finite_difference_jacobian_(J, f, x, cache))
        else:
            pkg.finite_difference_jacobian_(J, f, x, cache)
            torch.cuda.synchronize()
            kernels = []
    assert_same_bits(x, xh, f"{desc}: the caller's x", allow_nan=False)
    plan = cache._last_plan
    r = oracle.jacobian_complex(P, ref, oracle.native_fn("synth_ellrows_c"), xh.copy(), colorvec=cv, ctx=ell.octx(oracle))
    assert ctx.calls == r["fcalls"] == plan.info()["fcalls_per_jacobian"], (desc, ctx.calls, r["fcalls"])
    assert_same_bits(plan.eps(), np.full(r["fcalls"], EPS), f"{desc}: eps(Float64) for every colour", allow_nan=False)
    assert_same_bits(vals, ref, desc, allow_nan=False)
    only_complex_scatters(kernels, desc)
    return kernels, plan


# ------------------------------------------------------------------------------------------------ the synthetic f! itself
def test_synth_ellrows_c_matches_oracle(pkg, oracle, dev):
    """fdbs_ellrows_c == synth_ellrows_c bit for bit: a batch of 3 complex points (grid.y), padded ldx / ldfx."""
    rng = np.random.default_rng(1)
    m, n, K, B = 1500, 777, 5, 3
    ldx, ldfx = n + 3, m + 5
    ell = random_ell(dev, rng, m, n, K)
    X = np.full((B, ldx), NAN + 1j * NAN)    # the padding is never read
    X[:, :n] = make_x(rng, (B, n)) + 1j * np.where(rng.random((B, n)) < 0.3, rng.uniform(-1, 1, (B, n)), 0.0)
    X[1, :n].imag = np.where(np.arange(n) % 5 == 0, EPS, 0.0)
    d_X = torch.from_numpy(X).to(dev)
    d_F = torch.empty((B, ldfx), dtype=torch.complex128, device=dev)
    torch.view_as_real(d_F).fill_(NAN)
    f, ctx = ell.native(pkg)
    assert pkg._lib.synth().fdbs_ellrows_c(C.byref(ctx), d_F.data_ptr(), d_X.data_ptr(), B, ldfx, ldx, None) == 0
    torch.cuda.synchronize()
    assert ctx.calls == B
    F = torch.view_as_real(d_F).cpu().numpy()
    pd = C.POINTER(C.c_double)
    for b in range(B):
        x = np.ascontiguousarray(X[b, :n])
        ref = np.full(m, NAN + 1j * NAN)
        oracle.lib().synth_ellrows_c(C.byref(ell.octx(oracle)), ref.ctypes.data_as(pd), x.ctypes.data_as(pd))
        assert_same_bits(F[b, :m].reshape(-1), ref.view(np.float64), f"point {b}", allow_nan=False)
        re, im = ell_c_numpy(ell.cols, ell.coef, x)
        assert_same_bits(ref.real.copy(), re, allow_nan=False)
        assert_same_bits(ref.imag.copy(), im, allow_nan=False)
        assert np.isnan(F[b, m:]).all(), "rows past m of the padded output must stay untouched"


# ------------------------------------------------------------------------------------------------ random CSC patterns
def _case(rng, pkg, oracle, dev, sm_count=None, lo=1, hi=400):
    m = int(rng.integers(lo, hi))
    n = int(rng.integers(lo, hi))
    K = int(rng.integers(1, 6))
    ell = random_ell(dev, rng, m, n, K)                          # random dependence, duplicates allowed
    colptr, rowval = csc_of(m, n, ell, rng, extra=int(rng.integers(0, m + 1)))   # ragged / empty columns, spurious entries
    ncol = int(rng.integers(1, 12))
    cv = rng.integers(0 if rng.random() < 0.3 else 1, ncol + 1, size=n).astype(np.int64)   # 0 = no valid colour
    if cv.max() < 1:
        cv[0] = 1
    opts = dict(strategy=int(rng.integers(0, 4)), max_batch=int(rng.integers(1, 4)))
    if rng.random() < 0.35:
        # a budget of a few complex slabs (16 bytes per row): several scatter groups per Jacobian
        opts["scratch_bytes"] = int(16 * (m + 2) * int(rng.integers(1, 4)) + 64)
    dense = rng.random() < 0.3 and m * n <= 4_000_000
    sp = J_csc(pkg, m, n, colptr, rowval, dev)
    if dense:
        J, vals = J_dense(pkg, m, n, dev)
        P = oracle.Problem.csc_to_dense(m, n, colptr, rowval)
    else:
        J, vals = sp, sp.nzval
        P = oracle.Problem.csc_same(m, n, colptr, rowval)
    desc = f"m={m} n={n} K={K} C={cv.max()} {opts} dense={dense} sm_count={sm_count}"
    run(pkg, oracle, dev, J, vals, P, ell, make_x(rng, n), cv=cv, sparsity=sp, plan_kw=opts, env=dict(SM_COUNT=sm_count),
        trace=False, desc=desc)


def test_random_patterns_bitexact(pkg, oracle, dev):
    rng = np.random.default_rng(20261016)
    for _ in range(120):
        _case(rng, pkg, oracle, dev)


@pytest.mark.parametrize("sm_count", [1, 3])
def test_random_patterns_bitexact_multiwave(pkg, oracle, dev, sm_count):
    rng = np.random.default_rng(20261016 + sm_count)
    for _ in range(60):
        _case(rng, pkg, oracle, dev, sm_count)


@pytest.mark.parametrize("sm_count", [1, 3])
def test_random_patterns_mid_size_multiwave(pkg, oracle, dev, sm_count):
    rng = np.random.default_rng(20261017 + sm_count)
    for _ in range(4):
        _case(rng, pkg, oracle, dev, sm_count, lo=10_000, hi=100_000)


# ------------------------------------------------------------------------------------------------ CSC scatter forms
# (name, PlanOpts strategy, complex slabs per scratch budget (None: all), dense J, environment, expected kernel + args)
CSC_FORMS = [
    ("ident_full", 1, None, False, {}, ("diff_scatter_ident", dict(a2=TRUE))),
    ("ident_groups", 1, 2, False, {}, ("diff_scatter_ident", dict(a2=FALSE))),
    ("dest_dense", 1, None, True, {}, ("diff_scatter_dest", {})),
    ("dest_dense_groups", 1, 3, True, {}, ("diff_scatter_dest", {})),
    ("cm_groups", 2, 2, False, {}, ("diff_scatter_cm", dict(a1="int"))),
    ("cm_dense", 2, 3, True, {}, ("diff_scatter_cm", dict(a1="long"))),
    ("cm_prefetch", 3, None, False, {"CM_PREFETCH": 1}, ("diff_scatter_cm", dict(a1="int"))),
]


@pytest.mark.parametrize("sm_count", [None, 1, 3])
@pytest.mark.parametrize("form", CSC_FORMS, ids=[f[0] for f in CSC_FORMS])
def test_csc_scatter_forms(pkg, oracle, dev, form, sm_count):
    name, strategy, slabs, dense, env, (kernel, args) = form
    rng = np.random.default_rng(len(name))
    m, n, K, Cc = 3001, 2500, 4, 7
    ell = random_ell(dev, rng, m, n, K)
    colptr, rowval = csc_of(m, n, ell, rng, extra=500)
    cv = colouring("zero", n, Cc, rng)
    cv[rng.integers(0, n, 40)] = rng.integers(1, Cc + 1, 40)     # not a valid distance-2 colouring either
    cv[0] = Cc
    opts = dict(strategy=strategy, max_batch=3)
    if slabs is not None:
        opts["scratch_bytes"] = 16 * (m + 1) * slabs + 64
    sp = J_csc(pkg, m, n, colptr, rowval, dev)
    if dense:
        J, vals = J_dense(pkg, m, n, dev)
        P = oracle.Problem.csc_to_dense(m, n, colptr, rowval)
    else:
        J, vals = sp, sp.nzval
        P = oracle.Problem.csc_same(m, n, colptr, rowval)
    k, _ = run(pkg, oracle, dev, J, vals, P, ell, make_x(rng, n), cv=cv, sparsity=sp, plan_kw=opts,
            env=dict(env, SM_COUNT=sm_count), desc=name)
    hits = expect(k, kernel, **args)
    expect(k, "perturb_complex")
    if slabs is not None:
        assert len(hits) == -(-Cc // slabs), f"{name}: one scatter launch per group"
    if name == "cm_prefetch":
        assert len(hits) == 1, "all colours' lists in one launch (the prefetch of the next colour's slab runs)"


# ------------------------------------------------------------------------------------------------ banded targets
# (name, m, n, l, u, target, colouring, expected band kernel); the ELL f reads only in-band columns
BAND_CASES = [
    ("narrow_data", 500, 500, 2, 3, "band", "cyclic", "diff_scatter_band"),
    ("narrow_dense", 480, 500, 3, 2, "dense", "table", "diff_scatter_band"),
    ("narrow_zero_tall", 503, 500, 4, 1, "band", "zero", "diff_scatter_band"),
    ("wide_flat", 900, 900, 40, 30, "band", "cyclic", "diff_scatter_band_flat"),
    ("wide_flat_short", 880, 900, 35, 40, "band", "zero", "diff_scatter_band_flat"),
    ("wide_offset_tall", 900, 850, 50, 20, "band_offset", "table", "diff_scatter_band_wide"),
    ("wide_dense", 700, 760, 33, 33, "dense", "cyclic", "diff_scatter_band_wide"),
    ("wide_dense_zero", 760, 700, 70, 12, "dense", "zero", "diff_scatter_band_wide"),
    ("wider_than_2049", 2600, 2600, 1100, 1100, "band", "zero", "diff_scatter_band_flat"),
]


@pytest.mark.parametrize("sm_count", [None, 1, 3])
@pytest.mark.parametrize("case", BAND_CASES, ids=[c[0] for c in BAND_CASES])
def test_banded_every_width(pkg, oracle, dev, case, sm_count):
    name, m, n, l, u, target, kind, kernel = case
    rng = np.random.default_rng(m + 7 * l + u)
    w = l + u + 1
    ell = band_ell(dev, rng, m, n, l, u, 4)
    cv = colouring(kind, n, 7, rng)
    sp = pkg.BandedMatrix(m, n, l, u, device=dev)
    if target == "dense":
        J, vals = J_dense(pkg, m, n, dev)
        P = oracle.Problem.banded_to_dense(m, n, l, u)
    else:
        off = int(target == "band_offset")
        vals = torch.full((w * n + off,), NAN, dtype=torch.float64, device=dev)[off:]   # offset: 8-byte aligned only
        J = sp = pkg.BandedMatrix(m, n, l, u, data=vals)
        P = oracle.Problem.banded(m, n, l, u)
    k, _ = run(pkg, oracle, dev, J, vals, P, ell, make_x(rng, n), cv=cv, sparsity=sp, env=dict(SM_COUNT=sm_count), desc=name)
    expect(k, kernel)
    expect(k, "perturb_complex", a0="CyclicColors" if kind == "cyclic" else "TableColors<unsigned char>")


# ------------------------------------------------------------------------------------------------ COO targets
def test_coo_tridiagonal_slots(pkg, oracle, dev):
    rng = np.random.default_rng(3)
    N = 1000
    i = np.arange(N)
    cols = np.stack([np.maximum(i - 1, 0), i, np.minimum(i + 1, N - 1)])
    ell = Ell(dev, cols, rng.uniform(-1, 1, (3, N)))
    J = pkg.Tridiagonal(N, device=dev)
    J.buf.fill_(NAN)
    rows, cc, slots = tridiagonal_coo(N)
    P = oracle.Problem.coo_to_slots(N, N, rows, cc, slots, 3 * N - 2)
    k, _ = run(pkg, oracle, dev, J, J.buf, P, ell, make_x(rng, N), cv=colouring("zero", N, 3, rng), sparsity=J, desc="tridiagonal")
    expect(k, "diff_scatter_dest")


def test_coo_dense_prototype(pkg, oracle, dev):
    rng = np.random.default_rng(4)
    m, n = 300, 250
    ell = random_ell(dev, rng, m, n, 3)
    proto = np.zeros((m, n))
    proto[np.tile(np.arange(m), 3), ell.cols.reshape(-1)] = 1.0
    proto[rng.integers(0, m, 200), rng.integers(0, n, 200)] = 1.0       # spurious entries
    rows, cols = oracle.findstructralnz_dense(proto)
    J, vals = J_dense(pkg, m, n, dev)
    P = oracle.Problem.coo_to_dense(m, n, rows, cols)
    k, _ = run(pkg, oracle, dev, J, vals, P, ell, make_x(rng, n), cv=colouring("table", n, 11, rng),
            sparsity=torch.from_numpy(proto).to(dev), plan_kw=dict(max_batch=2), desc="dense prototype")
    expect(k, "diff_scatter_dest")


# ------------------------------------------------------------------------------------------------ dense column branch
DENSE_CASES = [   # (m, n, max_batch, padding rows, sm_count)
    (2500, 300, 1, 0, None),
    (2500, 301, 7, 0, None),
    (700, 2049, 7, 0, 1),
    (300, 2050, 1, 0, 3),
    (2049, 2050, 7, 0, 3),
    (2100, 301, 7, 5, 1),
    (41, 300, 7, 7, None),
]


@pytest.mark.parametrize("m,n,batch,pad,sm_count", DENSE_CASES)
def test_dense_columns(pkg, oracle, dev, m, n, batch, pad, sm_count):
    rng = np.random.default_rng(m + n + batch)
    ell = random_ell(dev, rng, m, n, 4)
    J, vals = J_dense(pkg, m, n, dev, ld=m + pad, fill=7.25 if pad else NAN)
    P = oracle.Problem(oracle.SP_NONE, oracle.J_DENSE, m, n, ldJ=m + pad, j_len=(m + pad) * n)
    k, _ = run(pkg, oracle, dev, J, vals, P, ell, make_x(rng, n), plan_kw=dict(max_batch=batch), env=dict(SM_COUNT=sm_count),
            desc=f"dense m={m} n={n} batch={batch} ld={m + pad}")
    if pad:
        assert (vals.view(n, m + pad)[:, m:] == 7.25).all(), "padding rows between the columns do not belong to J"
    assert len(expect(k, "replicate_x_complex")) == 1
    assert len(expect(k, "set_components_complex")) == -(-n // batch)
    cols = expect(k, "diff_columns")
    assert len(cols) == -(-n // batch)
    if m > 2048 and sm_count is None:
        assert min(g for _, g in cols) >= 2, "several row blocks per column"


def test_dense_colorvec_leading_columns(pkg, oracle, dev):
    """sparsity=None with a colorvec: component color_i is perturbed for color_i in 1:maximum(colorvec) and J[:, color_i]
    written; the columns beyond maximum(colorvec) keep their previous contents (no fill_matrix!)."""
    rng = np.random.default_rng(6)
    m, n, mx = 400, 301, 230
    ell = random_ell(dev, rng, m, n, 4)
    cv = rng.integers(1, mx + 1, n).astype(np.int64)
    cv[17] = mx
    J, vals = J_dense(pkg, m, n, dev, fill=7.25)
    k, _ = run(pkg, oracle, dev, J, vals, oracle.Problem.dense(m, n), ell, make_x(rng, n), cv=cv, plan_kw=dict(max_batch=7),
            desc="dense colorvec")
    assert (vals.view(n, m)[mx:] == 7.25).all()
    expect(k, "diff_columns")


# ------------------------------------------------------------------------------------------------ colour-table widths
@pytest.mark.parametrize("ncolors,bits,ct", [(300, 16, "unsigned short"), (70_000, 32, "int")])
def test_wide_colour_tables(pkg, oracle, dev, ncolors, bits, ct):
    rng = np.random.default_rng(ncolors)
    m, n = 650, 600
    ell = random_ell(dev, rng, m, n, 3)
    colptr, rowval = csc_of(m, n, ell, rng, extra=100)
    cv = colouring("zero", n, ncolors, rng) if ncolors < n else rng.integers(0, ncolors + 1, n).astype(np.int64)
    cv[5] = ncolors
    sp = J_csc(pkg, m, n, colptr, rowval, dev)
    xh = make_x(rng, n)
    small = ncolors <= 65535
    k, plan = run(pkg, oracle, dev, sp, sp.nzval, oracle.Problem.csc_same(m, n, colptr, rowval), ell, xh, cv=cv,
                  sparsity=sp, plan_kw=dict(max_batch=4), trace=small, desc=f"C={ncolors}")
    assert plan.info()["color_bits"] == bits
    if not small:
        # a trace of the whole call would hold ~10^5 kernel records: read the instantiations from rank 0 of a 64-way colour
        # split of the same problem instead (the same colour table, 1/64 of the launches)
        x = torch.from_numpy(xh).to(dev)
        sp = J_csc(pkg, m, n, colptr, rowval, dev)
        cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device=dev), "complex", colorvec=cv, sparsity=sp,
                                  max_batch=4, rank=0, world=64, strategy=1)
        f, ctx = ell.native(pkg, 4)
        k = traced(lambda: pkg.finite_difference_jacobian_(sp, f, x, cache))
        assert cache._last_plan.info()["color_bits"] == bits and ctx.calls == cache._last_plan.info()["n_local_colors"]
        only_complex_scatters(k)
    nps = {t[1] for t, _ in expect(k, "perturb_complex", a0=f"TableColors<{ct}>")}
    assert "4" in nps, "batched points (several colours per perturbation pass)"
    expect(k, "diff_scatter_ident", a0=ct)


# ------------------------------------------------------------------------------------------------ alignment
def test_unaligned_x_and_nzval(pkg, oracle, dev):
    """x and nzval offset by one element (8-byte aligned only: j_aligned = 0, scalar stores)."""
    rng = np.random.default_rng(8)
    m, n = 2000, 1900
    ell = random_ell(dev, rng, m, n, 4)
    colptr, rowval = csc_of(m, n, ell, rng, extra=50)
    for opts in (dict(strategy=1), dict(strategy=1, scratch_bytes=16 * (m + 1) * 2 + 64), dict(strategy=2)):
        sp = J_csc(pkg, m, n, colptr, rowval, dev, offset=True)
        assert sp.nzval.data_ptr() % 16 == 8
        k, _ = run(pkg, oracle, dev, sp, sp.nzval, oracle.Problem.csc_same(m, n, colptr, rowval), ell, make_x(rng, n),
                cv=colouring("zero", n, 5, rng), sparsity=sp, plan_kw=opts, x_offset=True, desc=f"unaligned {opts}")
        expect(k, "perturb_complex")


# ------------------------------------------------------------------------------------------------ every f! argument
def ell_torch(cols, coef, fx, x):
    """synth_ellrows_c on torch's element-wise operations (separate kernels, nothing fused: the same roundings as numpy)
    on view_as_real parts; x, fx complex128 of shape (n,) / (m,) or (batch, n) / (batch, m)."""
    xr = torch.view_as_real(x)
    a, b = xr[..., 0], xr[..., 1]
    x0r, x0i = a[..., cols[0]], b[..., cols[0]]
    re, im = coef[0] * x0r, coef[0] * x0i
    for p in range(1, cols.shape[0]):
        re = re + coef[p] * a[..., cols[p]]
        im = im + coef[p] * b[..., cols[p]]
    re = re + 0.1 * (x0r * x0r - x0i * x0i)
    im = im + 0.1 * (x0r * x0i + x0r * x0i)
    fr = torch.view_as_real(fx)
    fr[..., 0] = re
    fr[..., 1] = im


@pytest.mark.parametrize("kind", ["csc", "banded", "dense"])
@pytest.mark.parametrize("batched", [False, True])
def test_every_f_argument(pkg, oracle, dev, kind, batched):
    """Every complex point handed to f!, in call order, equals the oracle's bit for bit (re and im)."""
    rng = np.random.default_rng(9)
    m, n, l, u = 42, 40, 2, 1               # m = n + l: the last row still meets the band
    ell = band_ell(dev, rng, m, n, l, u, 3) if kind == "banded" else random_ell(dev, rng, m, n, 3)
    cols_t, coef_t = ell.d_cols.to(torch.int64), ell.d_coef
    got = []

    def f(fx, x):
        got.extend(torch.view_as_real(x).reshape(-1, 2 * n).cpu().numpy())
        ell_torch(cols_t, coef_t, fx, x)

    f.batched = batched
    want = []

    def f_np(fx, x):
        want.append(x.view(np.float64).copy())
        re, im = ell_c_numpy(ell.cols, ell.coef, x)
        fx.real[:] = re
        fx.imag[:] = im

    xh = make_x(rng, n)
    x = torch.from_numpy(xh).to(dev)
    fx = torch.zeros(m, dtype=torch.float64, device=dev)
    cv = None
    if kind == "csc":
        colptr, rowval = csc_of(m, n, ell, rng, extra=10)
        cv = colouring("zero", n, 5, rng)
        J = sp = J_csc(pkg, m, n, colptr, rowval, dev)
        vals, P = sp.nzval, oracle.Problem.csc_same(m, n, colptr, rowval)
    elif kind == "banded":
        cv = colouring("cyclic", n, l + u + 1, rng)
        J = sp = pkg.BandedMatrix(m, n, l, u, device=dev)
        J.data.fill_(NAN)
        vals, P = J.data, oracle.Problem.banded(m, n, l, u)
    else:
        sp = None
        J, vals = J_dense(pkg, m, n, dev)
        P = oracle.Problem.dense(m, n)
    cache = pkg.JacobianCache(x, fx, "complex", colorvec=cv, sparsity=sp, max_batch=3 if batched else 1)
    pkg.finite_difference_jacobian_(J, f, x, cache)
    torch.cuda.synchronize()
    ref = np.full(vals.numel(), NAN)
    r = oracle.jacobian_complex(P, ref, f_np, xh.copy(), colorvec=cv)
    assert len(got) == len(want) == r["fcalls"]
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same_bits(g, w, f"{kind}: argument of f! call {i}", allow_nan=False)
    assert_same_bits(vals, ref, kind, allow_nan=False)
    assert_same_bits(x, xh, allow_nan=False)


# ------------------------------------------------------------------------------------------------ plan reuse and graphs
def test_plan_reuse_and_graph_replay(pkg, oracle, dev):
    rng = np.random.default_rng(10)
    m, n = 1500, 1400
    ell = random_ell(dev, rng, m, n, 4)
    colptr, rowval = csc_of(m, n, ell, rng, extra=100)
    cv = colouring("zero", n, 6, rng)
    P = oracle.Problem.csc_same(m, n, colptr, rowval)
    xs = [make_x(rng, n) for _ in range(2)]
    refs = []
    for xh in xs:
        ref = np.full(len(rowval), NAN)
        oracle.jacobian_complex(P, ref, oracle.native_fn("synth_ellrows_c"), xh.copy(), colorvec=cv, ctx=ell.octx(oracle))
        refs.append(ref)
    for use_graph in (False, True):
        sp = J_csc(pkg, m, n, colptr, rowval, dev)
        x = torch.from_numpy(xs[0]).to(dev)
        f, ctx = ell.native(pkg)
        cache = pkg.JacobianCache(x, torch.zeros(m, dtype=torch.float64, device=dev), "complex", colorvec=cv, sparsity=sp,
                                  use_graph=use_graph)
        for i in (0, 1, 0):
            x.copy_(torch.from_numpy(xs[i]))          # same buffer, new values: a replay must read them
            sp.nzval.fill_(NAN)
            pkg.finite_difference_jacobian_(sp, f, x, cache)
            torch.cuda.synchronize()
            assert_same_bits(sp.nzval, refs[i], f"use_graph={use_graph}, x #{i}", allow_nan=False)
        assert len(cache._plans) == 1, "one plan serves every call"
        assert cache._last_plan.counters()["jacobians"] == 3


# ------------------------------------------------------------------------------------------------ ownership on one GPU
@pytest.mark.parametrize("strategy,kernel", [(1, "diff_scatter_ident"), (2, "diff_scatter_cm")])
def test_csc_two_ranks_into_one_j(pkg, oracle, dev, strategy, kernel):
    """world = 2 plans (rank 0 and 1, shared_j) store into one zero-filled J one after the other: the result is the
    unsharded complex J.  Rank 0 also writes the entries of columns without a valid colour."""
    L = pkg._lib
    lib = L.lib()
    rng = np.random.default_rng(11 + strategy)
    m, n, Cc = 1200, 1000, 9
    ell = random_ell(dev, rng, m, n, 4)
    colptr, rowval = csc_of(m, n, ell, rng, extra=200)
    cv = colouring("zero", n, Cc, rng)
    xh = make_x(rng, n)
    x = torch.from_numpy(xh).to(dev)
    ref = np.full(len(rowval), NAN)
    r = oracle.jacobian_complex(oracle.Problem.csc_same(m, n, colptr, rowval), ref, oracle.native_fn("synth_ellrows_c"),
                                xh.copy(), colorvec=cv, ctx=ell.octx(oracle))
    entry_colour = cv[np.repeat(np.arange(n), np.diff(colptr))]     # 0 = column without a valid colour
    Jsh = torch.zeros(len(rowval), dtype=torch.float64, device=dev)
    calls = 0
    for rank in (0, 1):
        o = L.PlanOpts(fdtype=L.FDB_COMPLEX, device=0, rank=rank, world=2, shared_j=1, strategy=strategy)
        h = C.c_void_p()
        L.check(lib.fdb_plan_create_csc(C.byref(h), m, n, colptr.ctypes.data, rowval.ctypes.data, L.FDB_J_CSC_NZVAL, None,
                                        None, 0, cv.ctypes.data, C.byref(o)))
        plan = pkg.Plan(h.value)
        f, ctx = ell.native(pkg)
        k = traced(lambda: L.check(lib.fdb_jacobian_complex(plan.handle, C.c_void_p(f.address), f.ctx_ptr, x.data_ptr(),
                                                             Jsh.data_ptr(), None)))
        info = plan.info()
        assert 0 < info["n_local_colors"] < Cc and ctx.calls == info["n_local_colors"]
        assert_same_bits(plan.eps(), np.full(Cc, EPS), allow_nan=False)
        expect(k, kernel, **({"a2": FALSE} if kernel == "diff_scatter_ident" else {}))
        only_complex_scatters(k)
        calls += ctx.calls
        # the same plan into a NaN-filled J: exactly this rank's entries are defined (rank 0 also owns the entries of
        # columns without a valid colour, which it sets to 0)
        Jr = torch.full((len(rowval),), NAN, dtype=torch.float64, device=dev)
        L.check(lib.fdb_jacobian_complex(plan.handle, C.c_void_p(f.address), f.ctx_ptr, x.data_ptr(), Jr.data_ptr(), None))
        got = Jr.cpu().numpy()
        owner = np.append(plan.color_owner(), 0)[entry_colour - 1]   # colour 0 -> index -1 -> rank 0
        mine = owner == rank
        assert_same_bits(got[mine], ref[mine], f"rank {rank}: its own entries", allow_nan=False)
        assert np.isnan(got[~mine]).all(), f"rank {rank} wrote entries it does not own"
    assert calls == r["fcalls"] == Cc
    assert_same_bits(Jsh, ref, "two ranks == unsharded", allow_nan=False)
    assert_same_bits(x, xh, allow_nan=False)


def test_dense_column_blocks_three_ranks(pkg, oracle, dev):
    L = pkg._lib
    lib = L.lib()
    rng = np.random.default_rng(12)
    m, n = 500, 301
    ell = random_ell(dev, rng, m, n, 4)
    xh = make_x(rng, n)
    x = torch.from_numpy(xh).to(dev)
    ref = np.full(m * n, NAN)
    oracle.jacobian_complex(oracle.Problem.dense(m, n), ref, oracle.native_fn("synth_ellrows_c"), xh.copy(), ctx=ell.octx(oracle))
    parts, end = [], 0
    for rank in range(3):
        o = L.PlanOpts(fdtype=L.FDB_COMPLEX, device=0, max_batch=7, rank=rank, world=3)
        h = C.c_void_p()
        L.check(lib.fdb_plan_create_dense(C.byref(h), m, n, m, C.byref(o)))
        plan = pkg.Plan(h.value)
        b, e = plan.dense_range()
        assert b == end and e > b
        end = e
        slab = torch.full((m * (e - b),), NAN, dtype=torch.float64, device=dev)
        f, ctx = ell.native(pkg)
        k = traced(lambda: L.check(lib.fdb_jacobian_complex(plan.handle, C.c_void_p(f.address), f.ctx_ptr, x.data_ptr(),
                                                             slab.data_ptr(), None)))
        assert ctx.calls == e - b
        assert_same_bits(plan.eps(), np.full(e - b, EPS), allow_nan=False)
        expect(k, "diff_columns")
        parts.append(slab)
    assert end == n
    assert_same_bits(torch.cat(parts), ref, "column blocks == unsharded", allow_nan=False)
    assert_same_bits(x, xh, allow_nan=False)


# ------------------------------------------------------------------------------------------------ entry points
def test_entry_point_errors(pkg, dev):
    L = pkg._lib
    lib = L.lib()
    rng = np.random.default_rng(13)
    m = n = 64
    ell = random_ell(dev, rng, m, n, 2)
    colptr, rowval = csc_of(m, n, ell, rng)
    cv = colouring("cyclic", n, 4, rng)
    x = torch.from_numpy(make_x(rng, n)).to(dev)
    J = torch.full((len(rowval),), NAN, dtype=torch.float64, device=dev)
    f, ctx = ell.native(pkg)
    fptr = C.c_void_p(f.address)

    def plan(fdtype):
        h = C.c_void_p()
        o = L.PlanOpts(fdtype=fdtype, device=0)
        L.check(lib.fdb_plan_create_csc(C.byref(h), m, n, colptr.ctypes.data, rowval.ctypes.data, L.FDB_J_CSC_NZVAL, None,
                                        None, 0, cv.ctypes.data, C.byref(o)))
        return pkg.Plan(h.value)

    pc, pf = plan(L.FDB_COMPLEX), plan(L.FDB_FORWARD)
    st = lib.fdb_jacobian(pc.handle, fptr, f.ctx_ptr, x.data_ptr(), J.data_ptr(), None, None, NAN, NAN, 1.0, None)
    assert st == L.FDB_ERR_INVALID and b"fdb_jacobian_complex" in lib.fdb_last_error()
    st = lib.fdb_jacobian_complex(pf.handle, fptr, f.ctx_ptr, x.data_ptr(), J.data_ptr(), None)
    assert st == L.FDB_ERR_INVALID
    g = C.c_void_p()
    devs = (C.c_int * 1)(0)
    o = L.PlanOpts(fdtype=L.FDB_COMPLEX, device=0)
    L.check(lib.fdb_group_create_csc(C.byref(g), 1, devs, m, n, colptr.ctypes.data, rowval.ctypes.data, L.FDB_J_CSC_NZVAL,
                                     None, None, 0, cv.ctypes.data, C.byref(o)))
    try:
        st = lib.fdb_group_jacobian(g, fptr, None, x.data_ptr(), J.data_ptr(), None, None, NAN, NAN, 1.0, None)
        assert st == L.FDB_ERR_UNSUPPORTED
    finally:
        lib.fdb_group_destroy(g)
    torch.cuda.synchronize()
    assert ctx.calls == 0 and torch.isnan(J).all(), "a refused call evaluates nothing and leaves J alone"
