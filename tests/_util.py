"""Shared helpers for the parity tests: pattern builders in the reference's (Julia) conventions —
Int64, 1-based CSC exactly as SparseMatrixCSC stores it."""
import contextlib
import os

import numpy as np
import scipy.sparse as sp


def _host_f64(a):
    if hasattr(a, "detach"):                     # torch tensor, on any device
        a = a.detach().cpu().numpy()
    a = np.asarray(a)
    assert a.dtype == np.float64, f"assert_same_bits compares float64 data, got {a.dtype}"
    return np.ascontiguousarray(a).reshape(-1)


def assert_same_bits(got, ref, what="", *, allow_nan=True):
    """Bit-for-bit equality of two float64 arrays (numpy arrays or torch tensors, CUDA ones included).

    The values are compared as uint64 bit patterns, so +0.0 and -0.0 differ (`==` and np.array_equal treat them as
    equal).  Every NaN counts as one class, whatever its sign and payload: the CPU and the GPU encode the NaNs they
    produce differently.  allow_nan=False also fails on any NaN, as np.array_equal without equal_nan does (for results
    that must be NaN-free, e.g. a J buffer pre-filled with NaN that every slot has to overwrite).  On a mismatch the
    message names the first differing index and both hex patterns."""
    g, r = _host_f64(got), _host_f64(ref)
    assert g.shape == r.shape, f"{what}: shapes differ, {g.shape} vs {r.shape}"
    if not allow_nan:
        assert not (np.isnan(g).any() or np.isnan(r).any()), f"{what}: NaN where none is expected"
    gb, rb = g.view(np.uint64), r.view(np.uint64)
    gn, rn = np.isnan(g), np.isnan(r)
    bad = np.flatnonzero((gb != rb) & ~(gn & rn))
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.size} of {g.size} values differ in their bits; first at index {i}: "
                             f"got {g[i]!r} (0x{int(gb[i]):016x}), expected {r[i]!r} (0x{int(rb[i]):016x})")


@contextlib.contextmanager
def fdb_env(**switches):
    """Set FDB_* switches (DESIGN.md §4) while plans are created, restoring the previous environment afterwards.
    fdb_env(NO_BAND=1, SM_COUNT=3) sets FDB_NO_BAND=1 and FDB_SM_COUNT=3; a value of None leaves the variable unset.
    Plans read the switches once, when they are created (for the Python mirror: on the first call that needs the plan)."""
    names = {f"FDB_{k}": v for k, v in switches.items()}
    saved = {k: os.environ.get(k) for k in names}
    try:
        for k, v in names.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def band_csc(m, n, l, u):
    """colptr/rowval (1-based Int64) of the clipped band: column c holds rows max(0, c-l) .. min(m-1, c+u)."""
    c = np.arange(n)
    lo, hi = np.maximum(c - l, 0), np.minimum(c + u, m - 1)
    cnt = np.maximum(hi - lo + 1, 0)
    colptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    rowval = np.arange(colptr[-1], dtype=np.int64) - np.repeat(colptr[:-1], cnt) + np.repeat(lo, cnt)
    return colptr + 1, rowval + 1


def tridiag_csc(n):
    """colptr/rowval (1-based Int64) of the n x n tridiagonal pattern (sparse(second_derivative_stencil))."""
    A = sp.diags([np.ones(n - 1), np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csc")
    A.sort_indices()
    return (A.indptr.astype(np.int64) + 1), (A.indices.astype(np.int64) + 1)


def csc_from_dense_pattern(A):
    S = sp.csc_matrix(np.asarray(A) != 0)
    S.sort_indices()
    return S.indptr.astype(np.int64) + 1, S.indices.astype(np.int64) + 1


def csc_to_dense(m, n, colptr, rowval, nzval):
    J = np.zeros((m, n))
    for c in range(n):
        for p in range(colptr[c] - 1, colptr[c + 1] - 1):
            J[rowval[p] - 1, c] = nzval[p]
    return J


def band_to_dense(m, n, l, u, data):
    """BandedMatrices storage data[(l+u+1) x n] column-major flat -> dense."""
    w = l + u + 1
    J = np.zeros((m, n))
    for c in range(1, n + 1):
        for r in range(max(1, c - u), min(m, c + l) + 1):
            J[r - 1, c - 1] = data[(c - 1) * w + (u + r - c)]
    return J


def cyc_colors(n, C):
    return (np.arange(n, dtype=np.int64) % C) + 1


def f_tridiag(dx, x):
    # test/coloring_tests.jl:5-13
    n = len(x)
    dx[1:n - 1] = (x[0:n - 2] - 2 * x[1:n - 1]) + x[2:n]
    dx[0] = -2 * x[0] + x[1]
    dx[n - 1] = x[n - 2] - 2 * x[n - 1]


def ell_c_numpy(cols, coef, x):
    """oracle/synth_fns.c:synth_ellrows_c restated on numpy's separate real operations (each one IEEE-rounded, nothing
    fused), in the same order: f_i = sum_p coef[p,i]*x[cols[p,i]] + 0.1*x0^2 on (re, im), x0 = x[cols[0,i]].
    cols, coef: ELL layout [K][m]; x: complex128.  Returns (re, im)."""
    a, b = x.real.copy(), x.imag.copy()
    x0r, x0i = a[cols[0]], b[cols[0]]
    re, im = coef[0] * x0r, coef[0] * x0i
    for p in range(1, cols.shape[0]):
        re = re + coef[p] * a[cols[p]]
        im = im + coef[p] * b[cols[p]]
    re = re + 0.1 * (x0r * x0r - x0i * x0i)
    im = im + 0.1 * (x0r * x0i + x0r * x0i)
    return re, im


def max_julia(a, b):
    """Julia's max on Float64: NaN propagates (as a - b), otherwise b when a - b is negative (so max(-0.0, 0.0) = 0.0)."""
    if np.isnan(a) or np.isnan(b):
        return np.float64(a - b)
    return b if np.signbit(np.float64(a - b)) else a


def hessian_transcribed(f, x, relstep=None, absstep=None):
    """hessians.jl:202-292, one Python line per Julia line (numpy float64 scalars: IEEE, one rounding per operation).
    Returns (H, f(x), every point f was called with)."""
    f64 = np.float64
    relstep = f64(2.0 ** -13) if relstep is None else f64(relstep)
    absstep = relstep if absstep is None else f64(absstep)
    points = []

    def F(v):
        points.append(v.copy())
        return f64(f(v.copy()))

    n = len(x)
    H = np.zeros((n, n))
    fx = F(x)
    xpp, xpm, xmp, xmm = x.copy(), x.copy(), x.copy(), x.copy()
    with np.errstate(all="ignore"):
        for i in range(n):
            xi = x[i]
            epsilon = max_julia(relstep * abs(xi), absstep)
            xpp[i] = xi + epsilon
            xmm[i] = xi - epsilon
            a = F(xpp)
            b = F(xmm)
            H[i, i] = (a - f64(2) * fx + b) / (epsilon * epsilon)
            epsiloni = max_julia(relstep * abs(xi), absstep)
            xp = xi + epsiloni
            xm = xi - epsiloni
            xpp[i], xpm[i], xmp[i], xmm[i] = xp, xp, xm, xm
            for j in range(i + 1, n):
                xj = x[j]
                epsilonj = max_julia(relstep * abs(xj), absstep)
                xp = xj + epsilonj
                xm = xj - epsilonj
                xpp[j], xpm[j], xmp[j], xmm[j] = xp, xm, xp, xm
                a, b, c, d = F(xpp), F(xpm), F(xmp), F(xmm)
                H[i, j] = (a - b - c + d) / (f64(4) * epsiloni * epsilonj)
                xpp[j], xpm[j], xmp[j], xmm[j] = xj, xj, xj, xj
            xpp[i], xpm[i], xmp[i], xmm[i] = xi, xi, xi, xi
        for i in range(n):
            for j in range(i + 1, n):
                H[j, i] = H[i, j]
    return H, fx, points


def gradient_transcribed(f, x, fdtype, fx=None, relstep=None, absstep=None, dir=1.0):
    """gradients.jl:390-457 (real x, real df; fdtype 0 forward, 1 central), one Python line per Julia line.
    Returns (df, every point f was called with)."""
    f64 = np.float64
    eps = np.finfo(float).eps
    if relstep is None:
        relstep = f64(np.sqrt(eps)) if fdtype == 0 else f64(np.cbrt(eps))
    absstep = relstep if absstep is None else f64(absstep)
    relstep = f64(relstep)
    points = []

    def F(v):
        points.append(v.copy())
        return f64(f(v.copy()))

    n = len(x)
    df = np.zeros(n)
    c3 = x.copy()
    with np.errstate(all="ignore"):
        if fdtype == 0:
            fx0 = f64(fx) if fx is not None else F(x)
            for i in range(n):
                epsilon = max_julia(relstep * abs(x[i]), absstep) * f64(dir)
                x_old = x[i]
                c3[i] += epsilon
                dfi = (F(c3) - fx0) / epsilon
                c3[i] = x_old
                df[i] = dfi
        else:
            for i in range(n):
                epsilon = max_julia(relstep * abs(x[i]), absstep)
                x_old = x[i]
                c3[i] += epsilon
                dfi = F(c3)
                c3[i] = x_old - epsilon
                dfi -= F(c3)
                c3[i] = x_old
                df[i] = dfi / (f64(2) * epsilon)
    return df, points


def blocked_sum(t):
    """Sum of the float64 vector t in the blocked order of the synthetic scalar functions (fdbs_quartic and its twins):
    1024-element blocks; lane l (of 32) adds elements l, l+32, ..., l+992 of its block in ascending order, starting from
    0.0 (0.0 past the end); an xor butterfly s[l] = s[l] + s[l ^ o], o = 16, 8, 4, 2, 1; block sums added in block order."""
    t = np.asarray(t, dtype=np.float64)
    nblk = -(-t.size // 1024)
    T = np.zeros(nblk * 1024)
    T[:t.size] = t
    T = T.reshape(nblk, 32, 32)                       # [block, j, lane] = element block*1024 + 32 j + lane
    s = np.zeros((nblk, 32))
    for j in range(32):
        s = s + T[:, j, :]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    S = np.float64(0.0)
    for b in range(nblk):
        S = S + s[b, 0]
    return S


def _guard(t, c):
    return np.where(np.isfinite(t) & (np.abs(t) <= 2.0 ** 500), t, np.float64(c))


def guarded_numpy(x, a, w):
    """fdbs_guarded (include/fdjac_synth.h) evaluated with numpy, independently of its C twin synth_guarded:
    f = sum_i (g(a_i x_i^4, 1/4) + g(x_i x_{i+1}, -1/2) + z_i) + s^2 / (2n), s = g(sum_i g(w_i x_i, 3/4), 3/2),
    z_i = (!isnan(x_i) && signbit(x_i)) ? w_i : 0, g(t, c) = (isfinite(t) && |t| <= 2^500) ? t : c."""
    x = np.asarray(x, dtype=np.float64)
    n = x.size
    with np.errstate(all="ignore"):
        q = x * x
        t1 = _guard(a * (q * q), 0.25)
        if n > 1:
            t1[:-1] = t1[:-1] + _guard(x[:-1] * x[1:], -0.5)
        t1 = t1 + np.where(~np.isnan(x) & np.signbit(x), w, 0.0)
        t2 = _guard(w * x, 0.75)
        S1, S2 = blocked_sum(t1), blocked_sum(t2)
        if n == 0:
            return S1
        s = np.float64(_guard(S2, 1.5))
        return S1 + (s * s) / np.float64(2 * n)


def exact_dot_xv(n, seed, kind="unit"):
    """x, v with x_j = a_j 2^-s and v_j = b_j 2^-t for integers |a_j| < 2^20, |b_j| < 2^12: for n <= 2^20 every product
    and every partial sum of dot(x, v) is a multiple of 2^-(s+t) below 2^53 * 2^-(s+t), so the dot is exact in any
    summation order and a device tree, the oracle's in-order loop and np.dot all give the same bits.
    kind: "unit" (s, t = 20, 12), "big" (x up to 2^500), "tiny" (d ~ 2^-950: the absstep branch of eps), "neg" (a
    negative dot), "zero" (pairs that cancel: the dot is exactly 0; needs even n for a +0.0 result)."""
    assert n <= 1 << 20
    rng = np.random.default_rng(seed)
    a = rng.integers(-(1 << 20) + 1, 1 << 20, n).astype(np.float64)
    b = rng.integers(-(1 << 12) + 1, 1 << 12, n).astype(np.float64)
    s, t = {"unit": (20, 12), "big": (-480, 12), "tiny": (500, 500), "neg": (20, 12), "zero": (20, 12)}[kind]
    if kind == "neg":
        b = -np.abs(b) * np.where(a < 0, -1.0, 1.0)
    if kind == "zero":
        a[1::2] = a[0:n - n % 2:2]
        b[1::2] = -b[0:n - n % 2:2]
        if n % 2:
            b[-1] = 0.0
    return np.ldexp(a, -s), np.ldexp(b, -t)


class GatherF:
    """A test f(fx, x) with m outputs of n inputs made only of gathers and separately rounded *, +, -:
    fx_i = (c_i * x[g0_i] + x[g1_i] * x[g2_i]) - d_i  (fx_i = -d_i when n = 0).  The numpy form (`np_f`) and the torch
    form (`torch_f`, one elementwise CUDA kernel per operation, so nothing is contracted into an FMA) round identically.
    Each form records a copy of every x it is called with."""

    def __init__(self, m, n, seed=0):
        rng = np.random.default_rng(seed + 7919 * m + n)
        self.m, self.n = m, n
        self.g = [rng.integers(0, max(n, 1), m) for _ in range(3)]
        self.c, self.d = rng.uniform(-2, 2, m), rng.uniform(-1, 1, m)

    def np_f(self, log):
        def f(fx, x):
            log.append(np.array(x, copy=True))
            with np.errstate(all="ignore"):
                if self.n == 0:
                    fx[:] = -self.d
                else:
                    fx[:] = (self.c * x[self.g[0]] + x[self.g[1]] * x[self.g[2]]) - self.d
        return f

    def torch_f(self, log, device):
        import torch
        g = [torch.from_numpy(i).to(device) for i in self.g]
        c, d = torch.from_numpy(self.c).to(device), torch.from_numpy(self.d).to(device)

        def f(fx, x):
            log.append(x.detach().cpu().numpy().copy())
            if self.n == 0:
                fx.copy_(-d)
            else:
                fx.copy_((c * x[g[0]] + x[g[1]] * x[g[2]]) - d)
        return f


def traced(fn):
    """Run fn() under torch.profiler (CUDA activity); return [(kernel name, grid x)] in launch order."""
    import json
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
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
    return [(e["name"], int(e.get("args", {}).get("grid", [1])[0]))
            for e in sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))]


def tridiagonal_coo(n):
    """Structural nz of Julia's Tridiagonal(dl,d,du) as (rows, cols, slots) with slots into [dl; d; du]
    (1-based): band order sub-diagonal, diagonal, super-diagonal."""
    rows = np.concatenate([np.arange(2, n + 1), np.arange(1, n + 1), np.arange(1, n)]).astype(np.int64)
    cols = np.concatenate([np.arange(1, n), np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int64)
    slots = np.arange(1, 3 * n - 1, dtype=np.int64)
    return rows, cols, slots


def tridiagonal_to_dense(n, buf):
    dl, d, du = buf[: n - 1], buf[n - 1: 2 * n - 1], buf[2 * n - 1:]
    return np.diag(d) + np.diag(dl, -1) + np.diag(du, 1)
