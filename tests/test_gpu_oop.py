"""The out-of-place Jacobian and JVP on the device (fdb_jacobian_oop / fdb_jacobian_oop_complex / fdb_jvp_oop, through the
Python mirror's finite_difference_jacobian / finite_difference_jvp) against the C restatement oop_oracle/ (itself held to the
line-by-line transcription tests/_literal_oop.py by tests/test_oop_oracle_cpu.py).

Every parity assert is a bit compare (assert_same_bits).  Coloured plans feed the restatement the step sizes the device
computed (the norm's summation order is not pinned), except where x's colour norms are exact; the dense branch and the complex step compute their own.  f is an
out-of-place torch function made of single IEEE operations (no fused kernels), and its numpy twin performs the same
operations in the same order, so both sides see bit-identical f values for bit-identical points.  Covered: every result
kind in forward, central and complex mode, dir = +-1 and 0.3, step overrides, f_in given or not, every point f sees in
order, the call count, sizes around the 1024-element tile, misaligned buffers, FDB_SM_COUNT 1 and 3 (with several tiles
per block of the new kernels, read from a profiler trace), the sparse result at C2 size with exactly-zero quotients on a
known subset, a dense result over 2 GB, plan reuse with x changed in place, cache.x1 after the call, the caller's x left
unchanged, and the rejections."""
import ctypes as C

import numpy as np
import pytest

import _literal_oop as LO
from oop_oracle import fd_oop_oracle as OO
from _util import assert_same_bits, fdb_env, traced, tridiag_csc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


# ---------------------------------------------------------------- f and its numpy twin
def _shift(x, lib):
    """(x[i-1], x[i+1]) with zeros past the ends"""
    if lib is np:
        z = np.zeros(1, dtype=x.dtype)
        return np.concatenate([z, x[:-1]]), np.concatenate([x[1:], z])
    z = torch.zeros(1, dtype=x.dtype, device=x.device)
    return torch.cat([z, x[:-1]]), torch.cat([x[1:], z])


def f_nl(x, lib=torch):
    """y_i = (x_i*x_i - 3*x_{i-1}) + (0.5*x_{i+1})*x_i : a tridiagonal, nonlinear f (real x only)"""
    xm, xp = _shift(x, lib)
    return (x * x - 3.0 * xm) + (0.5 * xp) * x


def f_lin(x, lib=torch):
    """y_i = (2*x_i + 3*x_{i-1}) - x_{i+1}: linear, so the complex step sees only products by real scalars"""
    xm, xp = _shift(x, lib)
    return (2.0 * x + 3.0 * xm) - xp


def f_masked(x, mask, lib=torch):
    """rows with mask 0 are constant (their quotients are +-0.0); row i reads x_i and x_{i+1}, not x_{i-1}, so the
    sub-diagonal quotients are +-0.0 too"""
    xm, xp = _shift(x, lib)
    return ((x * x) + 0.5 * xp) * mask + 1.0


class TorchF:
    """The out-of-place torch f, recording every point it is called with (as host copies when `record`)."""

    def __init__(self, fn, record=True):
        self.fn, self.record, self.points = fn, record, []

    def __call__(self, x):
        if self.record:
            self.points.append(x.detach().cpu().numpy().copy())
        return self.fn(x)


class NpF:
    def __init__(self, fn):
        self.fn, self.points = fn, []

    def __call__(self, x):
        self.points.append(np.array(x, copy=True))
        return self.fn(np.array(x, copy=True), np)


def _x(n, seed=0, zeros=True):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1.5, 1.5, n)
    if zeros and n > 3:
        x[1] = -0.0
        x[2] = 0.0
    return x


def _to_host_result(res):
    if isinstance(res, torch.Tensor):
        return ("dense", res.cpu().numpy())
    return ("sparse", res.m, res.n, res.colptr.cpu().numpy(), res.rowval.cpu().numpy(), res.nzval.cpu().numpy())


def assert_same_result(got, want, what=""):
    g = _to_host_result(got)
    assert g[0] == want[0], f"{what}: result kind {g[0]} != {want[0]}"
    if g[0] == "dense":
        assert_same_bits(g[1], want[1], f"{what}: J")
        return
    assert g[1:3] == tuple(want[1:3]), f"{what}: size {g[1:3]} != {want[1:3]}"
    assert np.array_equal(g[3], want[3]), f"{what}: colptr"
    assert np.array_equal(g[4], want[4]), f"{what}: rowval"
    assert_same_bits(g[5], want[5], f"{what}: nzval")


def _sparse_proto(pkg, m, n, colptr=None, rowval=None):
    if colptr is None:
        colptr, rowval = np.ones(n + 1, np.int64), np.zeros(0, np.int64)
    return pkg.SparseMatrixCSC(m, n, torch.from_numpy(colptr), torch.from_numpy(rowval),
                               torch.zeros(len(rowval), dtype=torch.float64, device="cuda"))


KINDS = ["raw", "dense_proto", "sparse_proto", "csc_dense", "csc_sparse"]


def _setup(pkg, kind, n, m=None):
    """(torch kwargs, literal kwargs) of a result kind on the tridiagonal pattern with cyclic colours 1:3"""
    m = n if m is None else m
    if kind in ("raw", "dense_proto", "sparse_proto"):
        if kind == "raw":
            return {}, {}
        if kind == "dense_proto":
            return ({"jac_prototype": torch.zeros((n + 1, m), dtype=torch.float64, device="cuda").t()},
                    {"jac_prototype": ("dense", m, n + 1)})
        return {"jac_prototype": _sparse_proto(pkg, m, n + 1)}, {"jac_prototype": ("sparse", m, n + 1)}
    cp, rv = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    tk = {"sparsity": S, "colorvec": cv}
    lk = {"sparsity": (n, n, cp, rv), "colorvec": cv}
    if kind == "csc_sparse":
        tk["jac_prototype"] = S
        lk["jac_prototype"] = ("sparse", n, n)
    return tk, lk


def _run(pkg, kind, fd, n, fn, x, *, dir=1.0, relstep=None, absstep=None, f_in=False, cacheless=False, record=True,
         cache_kw=None):
    """Device result + the transcription's, with every point each side's f saw."""
    tk, lk = _setup(pkg, kind, n)
    xd = torch.from_numpy(x).cuda()
    x_before = xd.clone()
    tf = TorchF(fn, record)
    fin_d = fn(xd) if f_in else None
    if cacheless:
        res = pkg.finite_difference_jacobian(tf, xd, fd, fin_d, relstep=relstep, absstep=absstep, dir=dir, **tk)
        cache = None
    else:
        cache = pkg.JacobianCache(xd, fd, **(cache_kw or {}))
        res = pkg.finite_difference_jacobian(tf, xd, cache, fin_d, relstep=relstep, absstep=absstep, dir=dir, **tk)
    torch.cuda.synchronize()
    assert_same_bits(xd, x_before, "the caller's x")
    rel = pkg.default_relstep(fd) if relstep is None else relstep
    # coloured plans: the device's step sizes (the cache-less form keeps no plan; its callers pass an x whose colour
    # norms are exact, so both sides compute the same steps)
    eps = list(cache._last_plan.eps()) if "sparsity" in lk and fd != "complex" and cache is not None else None
    nf = NpF(fn)
    want = OO.jacobian_oop(nf, x, fd, fn(x, np) if f_in else None, relstep=rel, absstep=absstep, dir=dir,
                           eps_override=eps, cacheless=cacheless, **lk)
    return res, want, tf, nf, cache


def _check_points(tf, nf, what):
    # the cache-less form's own f(x) is called by the mirror before the device call; both sides see it first
    assert len(tf.points) == len(nf.points), f"{what}: {len(tf.points)} calls, expected {len(nf.points)}"
    for i, (a, b) in enumerate(zip(tf.points, nf.points)):
        if np.iscomplexobj(b):
            assert_same_bits(np.real(a), np.real(b), f"{what}: point {i} (real)")
            assert_same_bits(np.imag(a), np.imag(b), f"{what}: point {i} (imag)")
        else:
            assert_same_bits(a, b, f"{what}: point {i}")


# ---------------------------------------------------------------- parity over kinds, modes, steps
CASES = []
for _fd in ("forward", "central"):
    for _dir in (1.0, -1.0, 0.3):
        for _steps in ((None, None), (1e-3, 0.0), (0.0, 1e-4)):
            CASES.append((_fd, _dir, _steps, False))
    CASES.append((_fd, 1.0, (None, None), True) if _fd == "forward" else (_fd, -1.0, (1e-2, None), False))
CASES.append(("complex", 1.0, (None, None), False))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fd,dir,steps,f_in", CASES)
@pytest.mark.parametrize("n", [7, 33])
def test_oop_jacobian_parity(pkg, kind, fd, dir, steps, f_in, n):
    fn = f_lin if fd == "complex" else f_nl
    x = _x(n, seed=n)
    if fd == "complex":
        x[1] = -0.0
    res, want, tf, nf, cache = _run(pkg, kind, fd, n, fn, x, dir=dir, relstep=steps[0], absstep=steps[1], f_in=f_in)
    what = f"{kind} {fd} dir={dir} steps={steps} f_in={f_in} n={n}"
    assert_same_result(res, want, what)
    _check_points(tf, nf, what)
    assert_same_bits(cache.x1.real if cache.x1.is_complex() else cache.x1, x, "cache.x1 after the call")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_oop_jacobian_cacheless_calls(pkg, kind, fd):
    n = 30
    fn = f_lin if fd == "complex" else f_nl
    x = np.random.default_rng(3).integers(-40, 40, n) * 2.0 ** -5      # exact colour norms
    res, want, tf, nf, _ = _run(pkg, kind, fd, n, fn, x, cacheless=True)
    assert_same_result(res, want, f"cache-less {kind} {fd}")
    _check_points(tf, nf, f"cache-less {kind} {fd}")
    C = 3 if kind.startswith("csc") else n
    assert len(tf.points) == 1 + (2 * C if fd == "central" else C)       # coloring_tests.jl:28-31: 31 at n = 30 forward


def test_oop_negative_zero_and_nan(pkg):
    n = 40
    mask = (np.arange(n) % 5 != 0).astype(np.float64)
    maskd = torch.from_numpy(mask).cuda()
    fn = lambda x, lib=torch: f_masked(x, mask if lib is np else maskd, lib)
    x = _x(n, seed=5)
    x[17] = np.nan
    for kind in KINDS:
        for dir in (1.0, -1.0):
            res, want, tf, nf, _ = _run(pkg, kind, "forward", n, fn, x, dir=dir)
            assert_same_result(res, want, f"masked {kind} dir={dir}")
            h = _to_host_result(res)
            if kind == "raw" and dir == -1.0:
                assert np.signbit(h[1][0, 0]) and h[1][0, 0] == 0         # -0.0 kept in the raw kind
            if kind in ("dense_proto", "csc_dense"):
                assert not (np.signbit(h[1]) & (h[1] == 0)).any()         # 0.0 + (-0.0): no -0.0 left
            if kind.endswith("sparse") or kind == "sparse_proto":
                assert not (h[5] == 0).any() and np.isnan(h[5]).any()      # no +-0.0 kept, NaN kept


# ---------------------------------------------------------------- sizes, grids, alignment
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025])
@pytest.mark.parametrize("sm", [None, 1, 3])
@pytest.mark.parametrize("kind", ["csc_sparse", "csc_dense", "sparse_proto", "dense_proto"])
def test_oop_tile_edges(pkg, n, sm, kind):
    if kind in ("sparse_proto", "dense_proto") and n > 1 and sm is not None and n != 1025:
        pytest.skip("dense branch: n calls of f; the grid switch is exercised at 1025")
    if kind.startswith("csc") and n < 3:
        kind_n = 3
    else:
        kind_n = n
    x = _x(kind_n, seed=kind_n)
    with fdb_env(SM_COUNT=sm):
        res, want, tf, nf, _ = _run(pkg, kind, "forward", kind_n, f_nl, x, dir=-1.0, record=kind_n < 64)
    assert_same_result(res, want, f"{kind} n={kind_n} sm={sm}")


def test_oop_empty_x_is_rejected(pkg):
    x = torch.zeros(0, dtype=torch.float64, device="cuda")
    with pytest.raises(pkg._lib.FdbError):
        pkg.finite_difference_jacobian(lambda v: v * 1.0, x, pkg.JacobianCache(x))


def test_oop_m_zero(pkg):
    x = torch.from_numpy(_x(5)).cuda()
    for proto in (None, "sparse"):
        kw = {} if proto is None else {"jac_prototype": _sparse_proto(pkg, 0, 5)}
        r = pkg.finite_difference_jacobian(lambda v: v[:0] * 1.0, x, pkg.JacobianCache(x, torch.zeros(0, dtype=torch.float64,
                                                                                                     device="cuda")), **kw)
        h = _to_host_result(r)
        if proto is None:
            assert h[1].shape == (0, 5)
        else:
            assert np.array_equal(h[3], np.ones(6, np.int64)) and h[4].size == 0


def test_oop_misaligned_inputs(pkg):
    n = 1030
    base = torch.from_numpy(np.concatenate([[7.0], _x(n, seed=9)])).cuda()
    xd = base[1:]                                      # 8 bytes past a 16-byte boundary
    x = xd.cpu().numpy()
    tk, lk = _setup(pkg, "csc_sparse", n)
    fbase = torch.zeros(n + 1, dtype=torch.float64, device="cuda")
    fin = fbase[1:]
    fin.copy_(f_nl(xd))
    cache = pkg.JacobianCache(xd, "forward")
    res = pkg.finite_difference_jacobian(TorchF(f_nl, False), xd, cache, fin, **tk)
    want = OO.jacobian_oop(NpF(f_nl), x, "forward", f_nl(x, np), eps_override=list(cache._last_plan.eps()), **lk)
    assert_same_result(res, want, "misaligned x and f_in")


def test_oop_misaligned_outputs_through_the_abi(pkg):
    """fdb_jacobian_oop with a dense J and with colptr / rowval / nzval 8 bytes past a 16-byte boundary"""
    L = pkg._lib
    n = 1500
    x = _x(n, seed=11)
    xd = torch.from_numpy(x).cuda()
    cp, rv = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    tf = TorchF(f_nl, False)
    addr, ctx, keep = pkg.api._as_fn(tf, n, n, xd.device, 1, oop=True)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    o = pkg.api._opts(L.FDB_FORWARD, 0)
    for kind in (L.FDB_OOP_DENSE, L.FDB_OOP_SPARSE):
        h = C.c_void_p()
        L.check(L.lib().fdb_oop_plan_create_csc(C.byref(h), n, n, cp.ctypes.data, rv.ctypes.data, cv.ctypes.data, kind, n,
                                                C.byref(o)))
        plan = pkg.Plan(h.value)
        out = L.OopOut()
        if kind == L.FDB_OOP_DENSE:
            Jb = torch.full((n * n + 1,), np.nan, dtype=torch.float64, device="cuda")
            out.J = Jb.data_ptr() + 8
        else:
            E = len(rv)
            cpb = torch.zeros(n + 2, dtype=torch.int64, device="cuda")
            rvb = torch.zeros(E + 1, dtype=torch.int64, device="cuda")
            nzb = torch.zeros(E + 1, dtype=torch.float64, device="cuda")
            nnz = torch.zeros(2, dtype=torch.int64, device="cuda")
            out.colptr, out.rowval, out.nzval, out.cap, out.nnz = (cpb.data_ptr() + 8, rvb.data_ptr() + 8,
                                                                   nzb.data_ptr() + 8, E, nnz.data_ptr() + 8)
        L.check(L.lib().fdb_jacobian_oop(plan.handle, addr, ctx, xd.data_ptr(), C.byref(out), None, None,
                                         L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, stream))
        torch.cuda.synchronize()
        eps = list(plan.eps())
        if kind == L.FDB_OOP_DENSE:
            want = OO.jacobian_oop(NpF(f_nl), x, "forward", sparsity=(n, n, cp, rv), colorvec=cv, eps_override=eps)
            got = Jb[1:].cpu().numpy().reshape(n, n).T
            assert_same_bits(got, want[1], "misaligned dense J")
            assert np.isnan(Jb[0].item())
        else:
            want = OO.jacobian_oop(NpF(f_nl), x, "forward", sparsity=(n, n, cp, rv), colorvec=cv, eps_override=eps,
                                   jac_prototype=("sparse", n, n))
            k = int(nnz[1].item())
            assert np.array_equal(cpb[1:].cpu().numpy(), want[3])
            assert np.array_equal(rvb[1:1 + k].cpu().numpy(), want[4])
            assert_same_bits(nzb[1:1 + k], want[5], "misaligned nzval")
            assert int(cpb[0].item()) == 0 and int(nnz[0].item()) == 0


def test_oop_new_kernels_take_several_tiles_per_block(pkg):
    n = 30000
    x = _x(n, seed=2)
    xd = torch.from_numpy(x).cuda()
    for kind in ("csc_sparse", "csc_dense"):
        tk, _ = _setup(pkg, kind, n)
        with fdb_env(SM_COUNT=1):
            cache = pkg.JacobianCache(xd, "forward")
            pkg.finite_difference_jacobian(TorchF(f_nl, False), xd, cache, **tk)   # plan built under the switch
        ev = traced(lambda: pkg.finite_difference_jacobian(TorchF(f_nl, False), xd, cache, **tk))
        name = "oop_compact" if kind == "csc_sparse" else "oop_plus_zero_slots"
        grids = [g for (k, g) in ev if name in k]
        assert grids, f"{name} not in the trace: {[k for k, _ in ev]}"
        E = 3 * n - 2
        per_block = (E + 1023) // 1024 if name == "oop_compact" else E / 256
        assert per_block / grids[0] >= 3, (name, grids[0], per_block)
    # oop_dense_finish: a dense prototype, m = 30000 rows from n = 8 components (30 row tiles x 9 columns)
    n8, rep_ = 8, 3750
    x8 = torch.from_numpy(_x(n8, seed=4)).cuda()
    f_wide = lambda v: (v * v).repeat(rep_)
    proto = torch.zeros((n8 + 1, n8 * rep_), dtype=torch.float64, device="cuda").t()
    with fdb_env(SM_COUNT=1):
        cache = pkg.JacobianCache(x8, "forward")
        pkg.finite_difference_jacobian(f_wide, x8, cache, jac_prototype=proto)
    ev = traced(lambda: pkg.finite_difference_jacobian(f_wide, x8, cache, jac_prototype=proto))
    grids = [g for (k, g) in ev if "oop_dense_finish" in k]
    assert grids and ((n8 * rep_ + 1023) // 1024) * (n8 + 1) / grids[0] >= 3, ev


# ---------------------------------------------------------------- plan reuse, C2 size, > 2 GB
def test_oop_plan_reuse_with_x_changed_in_place(pkg):
    n = 2000
    tk, lk = _setup(pkg, "csc_sparse", n)
    x = _x(n, seed=1)
    xd = torch.from_numpy(x).cuda()
    cache = pkg.JacobianCache(torch.zeros(n, dtype=torch.float64, device="cuda"), "central")
    for it in range(4):
        res = pkg.finite_difference_jacobian(TorchF(f_nl, False), xd, cache, dir=-1.0 if it % 2 else 1.0, **tk)
        want = OO.jacobian_oop(NpF(f_nl), x, "central", dir=-1.0 if it % 2 else 1.0,
                               eps_override=list(cache._last_plan.eps()), **lk)
        assert_same_result(res, want, f"reuse {it}")
        assert_same_bits(cache.x1, x, f"cache.x1 after call {it}")
        x = x * 1.25 + 0.5
        xd.copy_(torch.from_numpy(x))
    assert len(cache._plans) == 1


def test_oop_sparse_result_at_c2_size(pkg):
    """N = 10^7 tridiagonal, 3 colours, 3*10^7 candidate entries, f = the native stencil fdbs_tridiag, compared with the
    C restatement driving its CPU twin synth_tridiag (oracle/synth_fns.c).  Every 97th component is 2^90: each colour's
    step is then about 2^49 times relstep, below half an ulp of 2^90, so x + eps == x there and that column's quotients
    are exactly zero (dropped); the rows next to it lose their neighbours' steps in f ~ 2^91 too."""
    from oracle import fd_oracle as orc
    L = pkg._lib
    n = 10_000_000
    x = orc.fill_x(n, 0x5EED + 7)
    big = np.arange(5, n, 97)
    x[big] = 2.0 ** 90
    cp, rv = tridiag_csc(n)
    cv = (np.arange(n) % 3 + 1).astype(np.int64)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv),
                            torch.zeros(len(rv), dtype=torch.float64, device="cuda"))
    xd = torch.from_numpy(x).cuda()
    ctx = L.TridiagCtx(n, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
    twin = (C.cast(orc.native_fn("synth_tridiag"), C.c_void_p).value, orc.SynthTridiagCtx(n, 1))
    for fd, dir in (("forward", 1.0), ("central", -1.0)):
        cache = pkg.JacobianCache(xd, fd)
        res = pkg.finite_difference_jacobian(f, xd, cache, sparsity=S, colorvec=cv, jac_prototype=S, dir=dir)
        eps = list(cache._last_plan.eps())
        want = OO.jacobian_oop(twin, x, fd, sparsity=(n, n, cp, rv), colorvec=cv, jac_prototype=("sparse", n, n), dir=dir,
                               eps_override=eps)
        assert_same_result(res, want, f"C2 size {fd}")
        kept_cols = np.repeat(np.arange(n), np.diff(want[3]))
        assert not np.isin(kept_cols, big).any()                        # the 2^60 columns: every quotient dropped
        assert len(rv) // 2 < res.nnz < len(rv)


def test_oop_sparse_result_in_several_groups(pkg):
    """a scratch budget that holds one colour's f output at a time: the in-place scatter writes the candidates group by
    group and the compaction reads them (the form used when the outputs are not all resident)"""
    n = 5000
    x = _x(n, seed=8)
    tk, lk = _setup(pkg, "csc_sparse", n)
    xd = torch.from_numpy(x).cuda()
    for fd in ("forward", "central"):
        cache = pkg.JacobianCache(xd, fd, scratch_bytes=8 * (n + 2) * (2 if fd == "central" else 1))
        res = pkg.finite_difference_jacobian(TorchF(f_nl, False), xd, cache, dir=-1.0, **tk)
        assert cache._last_plan.info()["n_groups"] == 3
        want = OO.jacobian_oop(NpF(f_nl), x, fd, dir=-1.0, eps_override=list(cache._last_plan.eps()), **lk)
        assert_same_result(res, want, f"three groups {fd}")


@pytest.mark.parametrize("kind", ["csc_sparse", "csc_dense"])
@pytest.mark.parametrize("dir", [-1.0, 0.3])
def test_oop_coloured_central_step_takes_dir(pkg, kind, dir):
    """the coloured branch's central step is compute_epsilon(Val(:forward), sqrt(norm), ..., dir) (jacobians.jl:379-380):
    on x whose colour norms are exact the restatement computes its own step, so the sign and the factor of dir are
    checked, with every point f sees"""
    n = 40
    x = np.random.default_rng(21).integers(-40, 40, n) * 2.0 ** -5
    tk, lk = _setup(pkg, kind, n)
    xd = torch.from_numpy(x).cuda()
    tf, nf = TorchF(f_nl), NpF(f_nl)
    cache = pkg.JacobianCache(xd, "central")
    res = pkg.finite_difference_jacobian(tf, xd, cache, dir=dir, **tk)
    want = OO.jacobian_oop(nf, x, "central", dir=dir, **lk)
    assert_same_result(res, want, f"central {kind} dir={dir}")
    _check_points(tf, nf, f"central {kind} dir={dir}")
    rel = pkg.default_relstep("central")
    colours = np.arange(n) % 3 + 1
    for k in (1, 2, 3):
        norm = np.sqrt(np.sum(x[colours == k] ** 2))                     # exact sum of squares
        assert_same_bits([cache._last_plan.eps()[k - 1]], [LO.eps_forward(np.sqrt(norm), rel, rel, dir)], f"eps {k}")


@pytest.mark.parametrize("n,sm", [(341, None), (342, None), (342, 1), (343, 3), (683, None), (684, 1)])
def test_oop_compaction_tile_edges_in_entries(pkg, n, sm):
    """the compaction's tiles count candidates, E = 3n - 2 on the tridiagonal pattern: E = 1021, 1024 (the end pointer at
    position 1024 of the last tile), 1027, 2047, 2050"""
    x = _x(n, seed=n)
    with fdb_env(SM_COUNT=sm):
        res, want, tf, nf, _ = _run(pkg, "csc_sparse", "forward", n, f_nl, x, dir=-1.0, record=False)
    assert_same_result(res, want, f"E = {3 * n - 2}")


@pytest.mark.parametrize("n", [1023, 1024, 1025])
def test_oop_compaction_tile_edges_diagonal(pkg, n):
    """a diagonal sparsity: E = n candidates, one colour; every other entry's quotient is exactly zero"""
    x = _x(n, seed=n + 5)
    mask = (np.arange(n) % 2).astype(np.float64)
    maskd = torch.from_numpy(mask).cuda()
    fn = lambda v, lib=torch: (v * v) * (mask if lib is np else maskd) + 1.0
    cp, rv = np.arange(1, n + 2, dtype=np.int64), np.arange(1, n + 1, dtype=np.int64)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), torch.zeros(n, dtype=torch.float64,
                                                                                          device="cuda"))
    cv = np.ones(n, np.int64)
    xd = torch.from_numpy(x).cuda()
    cache = pkg.JacobianCache(xd, "forward")
    res = pkg.finite_difference_jacobian(TorchF(fn, False), xd, cache, sparsity=S, colorvec=cv, jac_prototype=S)
    want = OO.jacobian_oop(NpF(fn), x, "forward", sparsity=(n, n, cp, rv), colorvec=cv, jac_prototype=("sparse", n, n),
                           eps_override=list(cache._last_plan.eps()))
    assert_same_result(res, want, f"diagonal n={n}")
    assert res.nnz == n // 2


def test_oop_dense_result_over_2gb(pkg):
    n = 16400                                           # 16400^2 doubles = 2.15 GB
    x = _x(n, seed=6)
    tk, _ = _setup(pkg, "csc_dense", n)
    xd = torch.from_numpy(x).cuda()
    cache = pkg.JacobianCache(xd, "forward")
    J = pkg.finite_difference_jacobian(TorchF(f_nl, False), xd, cache, **tk)
    assert J.numel() * 8 > 2 * 2**30
    cp, rv = tridiag_csc(n)
    r0, c0, v = LO.jacobian_oop_csc_fast(lambda t: f_nl(t, np), x, "forward", list(cache._last_plan.eps()), n, cp, rv,
                                          np.arange(n) % 3 + 1, sparse=False)
    got = J[torch.from_numpy(r0).cuda(), torch.from_numpy(c0).cuda()]
    assert_same_bits(got, v, "structural slots")
    J[torch.from_numpy(r0).cuda(), torch.from_numpy(c0).cuda()] = 0.0
    assert int((J.view(torch.int64) != 0).sum().item()) == 0       # every other element +0.0


# ---------------------------------------------------------------- JVP
@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025])
@pytest.mark.parametrize("fd,dir,steps,f_in", [("forward", 1.0, (None, None), False), ("forward", -1.0, (1e-3, 0.0), True),
                                                ("forward", 0.3, (None, None), False), ("central", 1.0, (None, None), False),
                                                ("central", -1.0, (0.0, 1e-4), False)])
def test_oop_jvp(pkg, n, fd, dir, steps, f_in):
    x, v = _x(n, seed=n + 1), _x(n, seed=n + 2, zeros=False)
    xd, vd = torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda()
    x_before = xd.clone()
    tf = TorchF(f_nl)
    cache = pkg.JVPCache(xd, fd)
    fin = f_nl(xd) if f_in else None
    got = pkg.finite_difference_jvp(tf, xd, vd, cache, fin, relstep=steps[0], absstep=steps[1], dir=dir)
    torch.cuda.synchronize()
    e = float(cache._last_plan.eps()[0])
    nf = NpF(f_nl)
    want, _ = OO.jvp_oop(nf, x, v, fd, f_nl(x, np) if f_in else None, dir=dir, eps_override=e)
    assert_same_bits(got, want, f"jvp {fd} n={n}")
    _check_points(tf, nf, f"jvp {fd} n={n}")
    assert_same_bits(xd, x_before, "the caller's x")
    rel = pkg.default_relstep(fd) if steps[0] is None else steps[0]
    if n and np.dot(x, v) == 0.0:
        assert e == LO.eps_forward(0.0, rel, rel if steps[1] is None else steps[1], dir)


def test_oop_jvp_cacheless_and_exact_step(pkg):
    n = 64
    x = np.arange(1, n + 1) * 2.0 ** -4                 # x.v is exact in any summation order
    v = (np.arange(n) % 7 - 3) * 2.0 ** -3
    xd, vd = torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda()
    for fd in ("forward", "central"):
        tf, nf = TorchF(f_nl), NpF(f_nl)
        got = pkg.finite_difference_jvp(tf, xd, vd, fd, dir=-1.0)
        want, _ = OO.jvp_oop(nf, x, v, fd, dir=-1.0, cacheless=True)
        assert_same_bits(got, want, f"cache-less jvp {fd}")
        _check_points(tf, nf, f"cache-less jvp {fd}")


# ---------------------------------------------------------------- rejections
def test_oop_rejections(pkg):
    n = 6
    xd = torch.from_numpy(_x(n)).cuda()
    cache = pkg.JacobianCache(xd)
    f = lambda v: v * 1.0
    with pytest.raises(TypeError, match="not built"):
        pkg.finite_difference_jacobian(f, xd, cache, sparsity=pkg.Tridiagonal(n))
    with pytest.raises(TypeError, match="not built"):
        pkg.finite_difference_jacobian(f, xd, cache, jac_prototype=pkg.Tridiagonal(n))
    with pytest.raises(TypeError, match="not built"):
        pkg.finite_difference_jacobian(lambda v: v.to(torch.complex128), xd, cache)
    with pytest.raises(TypeError, match="not built"):
        pkg.finite_difference_jvp(lambda v: v.to(torch.complex128), xd, xd, pkg.JVPCache(xd))
    # a dense result on an invalid colouring: _make_Ji throws
    cp, rv = tridiag_csc(n)
    S = pkg.SparseMatrixCSC(n, n, torch.from_numpy(cp), torch.from_numpy(rv), torch.zeros(len(rv), dtype=torch.float64,
                                                                                          device="cuda"))
    bad = np.ones(n, np.int64)
    with pytest.raises(pkg._lib.FdbError, match="invalid colouring"):
        pkg.finite_difference_jacobian(f, xd, pkg.JacobianCache(xd), sparsity=S, colorvec=bad)
    # ... while the sparse result takes it, as the reference's sparse _make_Ji does
    r = pkg.finite_difference_jacobian(f, xd, pkg.JacobianCache(xd), sparsity=S, colorvec=bad, jac_prototype=S)
    assert r.nnz > 0
    # the in-place entry point refuses an out-of-place plan
    plan = pkg.JacobianCache(xd)
    pkg.finite_difference_jacobian(f, xd, plan, sparsity=S, colorvec=(np.arange(n) % 3 + 1))
    p = plan._last_plan
    with pytest.raises(pkg._lib.FdbError, match="out-of-place plan"):
        some_f = C.cast(pkg._lib.synth().fdbs_tridiag, C.c_void_p).value     # never called: the plan is refused first
        pkg._lib.check(pkg._lib.lib().fdb_jacobian(p.handle, some_f, None, xd.data_ptr(), xd.data_ptr(), None, None,
                                                   pkg._lib.STEP_DEFAULT, pkg._lib.STEP_DEFAULT, 1.0, None))
