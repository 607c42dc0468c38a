"""GPU parity on IEEE edge inputs (run with -m gpu on an H100): signed zeros, NaN and +-Inf in x.

Every case runs the device through the Python mirror with a Python f! that records each argument it is called with, and
the CPU oracle fed the device step sizes with the same f!.  Bars, bit for bit (_util.assert_same_bits: bit patterns,
every NaN one class): every f! argument, in call order; J.  The device's own step sizes are within rtol 1e-13 of the
oracle's (NaN where the oracle's are NaN).

f! is the tridiagonal stencil plus copysign(0.5, x_i), so the sign of a zero component changes f and J, not only the
bits of a zero: the reference adds eps_k*false = copysign(0, eps_k) to every component outside colour k (Julia's Bool
product is a strong zero), which turns a -0.0 into +0.0 from the first colour on."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

from _util import assert_same_bits, cyc_colors, fdb_env, tridiag_csc  # noqa: E402

FD = {"forward": 0, "central": 1}


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64))


def f_sign_np(dx, x):
    n = len(x)
    dx[1:n - 1] = (x[0:n - 2] - 2 * x[1:n - 1]) + x[2:n]
    dx[0] = -2 * x[0] + x[1]
    dx[n - 1] = x[n - 2] - 2 * x[n - 1]
    dx += np.copysign(0.5, x)


def f_sign_t(dx, x):                    # the same IEEE operations on CUDA tensors; 1-D or a (batch, n) block
    n = x.shape[-1]
    dx[..., 1:n - 1] = (x[..., 0:n - 2] - 2 * x[..., 1:n - 1]) + x[..., 2:n]
    dx[..., 0] = -2 * x[..., 0] + x[..., 1]
    dx[..., n - 1] = x[..., n - 2] - 2 * x[..., n - 1]
    dx += torch.copysign(torch.full_like(x, 0.5), x)


def recording_t(log, batched):
    def f(dx, x):
        log.extend(np.array(r, copy=True) for r in x.reshape(-1, x.shape[-1]).cpu().numpy())
        f_sign_t(dx, x)
    f.batched = batched
    return f


def recording_np(log):
    def f(dx, x):
        log.append(np.array(x, copy=True))
        f_sign_np(dx, x)
    return f


def x_with_zeros(N, seed):
    """Nonzero values of both signs, with -0.0 and +0.0 at the head (every colour), around the 1024-element tile
    boundaries and in the scalar tail."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.5, 2.0, N) * np.where(rng.random(N) < 0.5, -1.0, 1.0)
    idx = [i for i in [0, 1, 2, 3, 4, 5, 1021, 1022, 1023, 1024, 1025, 1026, 2047, 2048, 2049] if i < N]
    idx += list(range(max(0, N - 7), N))
    for t, i in enumerate(idx):
        x[i] = -0.0 if t % 2 == 0 else 0.0
    return x


def run_csc(pkg, oracle, dev, x_np, fdtype, cv, *, target="nzval", dir=1.0, no_drift=False, max_batch=1, sm_count=None,
            no_band=None, absstep=None, strategy=0, unaligned=False, scratch_bytes=0):
    N = len(x_np)
    colptr, rowval = tridiag_csc(N)
    xbuf = torch.zeros(N + 1, dtype=torch.float64, device=dev)
    x = xbuf[1:] if unaligned else xbuf[:N]
    x.copy_(torch.from_numpy(x_np))
    sp = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64,
                                                                          device=dev))
    if target == "dense":                # destination scatter: CSC sparsity into a dense column-major J
        J = pkg.zeros_colmajor(N, N, dev)
        J.fill_(float("nan"))
        P = oracle.Problem.csc_to_dense(N, N, colptr, rowval)
    else:
        J = sp
        P = oracle.Problem.csc_same(N, N, colptr, rowval)
    log = []
    f = recording_t(log, max_batch > 1)
    kw = {} if absstep is None else {"absstep": absstep}
    with fdb_env(SM_COUNT=sm_count, NO_BAND=no_band):
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=sp, no_drift=no_drift, max_batch=max_batch,
                                  strategy=strategy, scratch_bytes=scratch_bytes)
        pkg.finite_difference_jacobian_(J, f, x, cache, dir=dir, **kw)
    torch.cuda.synchronize()
    assert_same_bits(x, x_np, "the caller's x is never written")
    eps = cache._last_plan.eps()
    got = J.cpu().numpy().reshape(-1, order="F") if target == "dense" else sp.nzval.cpu().numpy()
    olog = []
    ref = np.zeros(N * N) if target == "dense" else np.full(len(rowval), np.nan)
    r = oracle.jacobian(P, ref, recording_np(olog), x_np.copy(), fdtype=FD[fdtype], colorvec=cv, eps_override=eps, dir=dir,
                        no_drift=no_drift, **kw)
    own = oracle.jacobian(P, np.zeros_like(ref), f_sign_np, x_np.copy(), fdtype=FD[fdtype], colorvec=cv, dir=dir, **kw)
    what = f"{fdtype} dir={dir} no_drift={no_drift} batch={max_batch} sm_count={sm_count} target={target}"
    if fdtype == "central" and max_batch > 1:
        # a batched f! gets the plus points of up to max_batch colours in one call, then their minus points; the
        # oracle calls plus, minus colour by colour
        pairs = [olog[i:i + 2] for i in range(0, len(olog), 2)]
        olog = [p[s] for i in range(0, len(pairs), max_batch) for s in (0, 1) for p in pairs[i:i + max_batch]]
    assert len(log) == len(olog) == r["fcalls"], what
    for i, (a, b) in enumerate(zip(log, olog)):
        assert_same_bits(a, b, f"{what}: argument of f! call {i}")
    assert_same_bits(got, ref, f"{what}: J")
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-13, atol=0)
    return dict(eps=eps, own=own["eps"], got=got, log=log)


def table_colors(N):
    """A valid distance-2 colouring of the tridiagonal pattern that is not cyclic: 3 colours repeated as 2,3,1, with a
    4th colour spliced in (the plan reads the colour table)."""
    cv = np.array([2, 3, 1], dtype=np.int64)[np.arange(N) % 3]
    cv[N // 2] = 4
    return cv


# ------------------------------------------------------------------------------------------------------- signed zeros
@pytest.mark.parametrize("colouring", ["cyclic", "table"])
@pytest.mark.parametrize("max_batch", [1, 4])
@pytest.mark.parametrize("no_drift", [False, True])
@pytest.mark.parametrize("fdtype,dir", [("forward", 1.0), ("forward", -1.0), ("central", 1.0)])
def test_signed_zeros_every_f_argument(pkg, oracle, dev, fdtype, dir, no_drift, max_batch, colouring):
    N = 3001
    cv = cyc_colors(N, 3) if colouring == "cyclic" else table_colors(N)
    r = run_csc(pkg, oracle, dev, x_with_zeros(N, 11), fdtype, cv, dir=dir, no_drift=no_drift, max_batch=max_batch)
    # component 2 is -0.0 in colour 3.  Forward: f(x) sees -0.0; colour 1 adds copysign(0, eps_1), which keeps -0.0 only
    # for dir = -1; after that whole colour it is +0.0, and colour 3 perturbs it to eps_3, which has the sign of dir.
    if colouring == "cyclic" and fdtype == "forward":
        assert [bool(np.signbit(a[2])) for a in r["log"]] == [True, dir < 0, False, dir < 0]


@pytest.mark.parametrize("fdtype,dir", [("forward", 1.0), ("forward", -1.0), ("central", 1.0)])
@pytest.mark.parametrize("max_batch", [1, 4])
@pytest.mark.parametrize("unaligned", [False, True])
def test_signed_zeros_multi_tile_and_unaligned(pkg, oracle, dev, fdtype, dir, max_batch, unaligned):
    # several 1024-element tiles per block (FDB_SM_COUNT=1), one point per launch and batches of 4, and an x that is only
    # 8-byte aligned (scalar paths).  Zeros sit in some full tiles; the others take the zero-free form of the kernel.
    N = 20_003
    for cv in (cyc_colors(N, 3), table_colors(N)):
        run_csc(pkg, oracle, dev, x_with_zeros(N, 12), fdtype, cv, dir=dir, sm_count=1, unaligned=unaligned,
                max_batch=max_batch)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_zero_colour_with_zero_absstep(pkg, oracle, dev, fdtype):
    # colour 2 all zeros of both signs and absstep = 0: eps_2 = 0 (-0.0 forward with dir = -1), J of that colour is
    # +-Inf or NaN, and the colour's own components see (+-0.0 or +0.0) +- 0.0 with the reference's signs
    N = 2051
    cv = cyc_colors(N, 3)
    x = x_with_zeros(N, 13)
    x[cv == 2] = np.where(np.arange((cv == 2).sum()) % 2, 0.0, -0.0)
    for dir in ((1.0, -1.0) if fdtype == "forward" else (1.0,)):
        r = run_csc(pkg, oracle, dev, x, fdtype, cv, dir=dir, absstep=0.0)
        assert r["eps"][1] == 0.0 and bool(np.signbit(r["eps"][1])) == (fdtype == "forward" and dir < 0)


@pytest.mark.parametrize("dir", [1.0, -1.0])
def test_zero_signs_of_J_entries(pkg, oracle, dev, dir):
    # f! constant: every difference is 1.0 - 1.0 = +0.0, and +0.0 / eps has the sign of eps, i.e. of dir
    N = 1000
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    x = torch.from_numpy(np.random.default_rng(14).uniform(1.0, 2.0, N)).to(dev)
    J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64,
                                                                        device=dev))
    pkg.finite_difference_jacobian_(J, lambda dx, xx: dx.fill_(1.0), x, pkg.JacobianCache(x, "forward", colorvec=cv,
                                                                                          sparsity=J), dir=dir)
    torch.cuda.synchronize()
    got = J.nzval.cpu().numpy()
    assert (got == 0.0).all() and (np.signbit(got) == (dir < 0)).all()


# ---------------------------------------------------------------------------------------------------------- NaN / Inf
def _bad_x(N, kind, cv, seed=21):
    x = np.random.default_rng(seed).uniform(-2, 2, N)
    c2 = np.flatnonzero(cv == 2)
    if kind == "nan":
        x[c2[len(c2) // 2]] = np.nan
    elif kind == "+inf":
        x[c2[len(c2) // 2]] = np.inf
    elif kind == "-inf":
        x[c2[len(c2) // 2]] = -np.inf
    elif kind == "nan_colour":
        x[c2] = np.nan
    return x


BAD = ["nan", "+inf", "-inf", "nan_colour"]
PATHS = [  # (name, run_csc keywords): the CSC formulations of the scatter
    ("staged_band", {}),
    ("staged_indexed", {"no_band": 1}),
    ("colour_major", {"strategy": 1}),
    ("column_lists", {"strategy": 2}),
    ("destination", {"target": "dense"}),
    ("gather", {"colors": 20}),                                   # more colours than the staged form takes: list ε pass
    ("gather_groups", {"colors": 20, "strategy": 1, "slabs": 2}),  # a two-slab budget: several groups (non-FULL)
]


@pytest.mark.parametrize("path", [p[0] for p in PATHS])
@pytest.mark.parametrize("bad", BAD)
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_nan_inf_in_x(pkg, oracle, dev, fdtype, bad, path):
    N = 2003 if path == "destination" else 5003          # the destination J is dense
    kw = dict(dict(PATHS)[path])
    cv = cyc_colors(N, kw.pop("colors", 3))
    if kw.pop("slabs", None):
        kw["scratch_bytes"] = 8 * (N + 2) * (4 if fdtype == "central" else 2) + 64
    r = run_csc(pkg, oracle, dev, _bad_x(N, bad, cv), fdtype, cv, **kw)
    e = r["eps"]
    others = np.delete(e, 1)
    assert np.isfinite(others).all()
    if bad.startswith("nan"):
        assert np.isnan(e[1])                                                  # Julia's max propagates NaN
    else:
        assert e[1] == np.inf


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("bad", BAD)
def test_nan_inf_in_x_banded(pkg, oracle, dev, fdtype, bad):
    N, l, u = 4000, 1, 1
    cv = cyc_colors(N, 3)
    x_np = _bad_x(N, bad, cv)
    x = torch.from_numpy(x_np).to(dev)
    Jb = pkg.BandedMatrix(N, N, l, u, device=dev)
    Jb.data.fill_(float("nan"))
    log = []
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=Jb)
    pkg.finite_difference_jacobian_(Jb, recording_t(log, False), x, cache)
    torch.cuda.synchronize()
    eps = cache._last_plan.eps()
    olog = []
    own = oracle.jacobian(oracle.Problem.banded(N, N, l, u), np.zeros((l + u + 1) * N), f_sign_np, x_np.copy(),
                          fdtype=FD[fdtype], colorvec=cv)
    ref = np.full((l + u + 1) * N, np.nan)
    oracle.jacobian(oracle.Problem.banded(N, N, l, u), ref, recording_np(olog), x_np.copy(), fdtype=FD[fdtype], colorvec=cv,
                    eps_override=eps)
    np.testing.assert_allclose(eps, own["eps"], rtol=1e-13, atol=0)
    assert len(log) == len(olog)
    for i, (a, b) in enumerate(zip(log, olog)):
        assert_same_bits(a, b, f"{fdtype} {bad}: argument of f! call {i}")
    assert_same_bits(Jb.data, ref, f"{fdtype} {bad}: band data")


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_nan_inf_in_x_dense_columns(pkg, oracle, dev, fdtype):
    # sparsity === nothing: per-component steps; NaN in x gives a NaN step (max propagates NaN), -0.0 a step of absstep
    N = 700
    x_np = np.random.default_rng(22).uniform(-2, 2, N)
    x_np[[3, 100, 101, 102, 699]] = [np.nan, np.inf, -np.inf, -0.0, 0.0]
    x = torch.from_numpy(x_np).to(dev)
    J = pkg.zeros_colmajor(N, N, dev)
    J.fill_(float("nan"))
    log = []
    cache = pkg.JacobianCache(x, torch.zeros(N, dtype=torch.float64, device=dev), fdtype)
    pkg.finite_difference_jacobian_(J, recording_t(log, False), x, cache)
    torch.cuda.synchronize()
    olog = []
    ref = np.zeros(N * N)
    r = oracle.jacobian(oracle.Problem.dense(N, N), ref, recording_np(olog), x_np.copy(), fdtype=FD[fdtype])
    assert np.isnan(r["eps"][3])
    assert_same_bits(cache._last_plan.eps(), r["eps"], "per-component steps")
    assert len(log) == len(olog)
    for i, (a, b) in enumerate(zip(log, olog)):
        assert_same_bits(a, b, f"argument of f! call {i}")
    assert_same_bits(J.cpu().numpy().reshape(-1, order="F"), ref, "J")


@pytest.mark.parametrize("bad", ["nan", "+inf", "signed_zeros"])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_edge_inputs_jvp(pkg, oracle, dev, fdtype, bad):
    # jvp.jl:252-253: sqrt(abs(dot(x, v))) is NaN for a NaN in x, and max(NaN, absstep) keeps it; Inf gives eps = Inf.
    # The device's f! arguments and output against the oracle's fed the device eps, bit for bit.
    N = 3000
    x_np = np.random.default_rng(23).uniform(-2, 2, N)
    v_np = np.random.default_rng(24).uniform(-1, 1, N)
    if bad == "nan":
        x_np[17] = np.nan
    elif bad == "+inf":
        x_np[17] = np.inf
    else:
        x_np = x_with_zeros(N, 25)
        v_np[::7] = -0.0
    x, v = torch.from_numpy(x_np).to(dev), torch.from_numpy(v_np).to(dev)
    jvp = torch.full((N,), float("nan"), dtype=torch.float64, device=dev)
    cache = pkg.JVPCache(x, fdtype)
    log, olog = [], []
    pkg.finite_difference_jvp_(jvp, recording_t(log, False), x, v, cache)
    torch.cuda.synchronize()
    eps = float(cache._last_plan.eps()[0])
    own = oracle.jvp(f_sign_np, x_np.copy(), v_np.copy(), N, fdtype=FD[fdtype])
    if bad == "nan":
        assert np.isnan(eps) and np.isnan(own["eps"])
    elif bad == "+inf":
        assert eps == own["eps"] == np.inf
    else:
        np.testing.assert_allclose(eps, own["eps"], rtol=1e-13)
    r = oracle.jvp(recording_np(olog), x_np.copy(), v_np.copy(), N, fdtype=FD[fdtype], eps_override=eps)
    assert len(log) == len(olog) == r["fcalls"]
    for i, (a, b) in enumerate(zip(log, olog)):
        assert_same_bits(a, b, f"{fdtype} {bad}: argument of f! call {i}")
    assert_same_bits(jvp, r["jvp"], f"{fdtype} {bad}: jvp")


# ------------------------------------------------------------------------------------------------------- complex step
@pytest.mark.parametrize("dense", [False, True])
def test_signed_zeros_complex_step(pkg, oracle, dev, dense):
    # x1 .+ im*eps .* (colour .== k) adds (+0.0, eps) or (+0.0, +0.0): the real part of every component is x + 0.0.
    # The dense-column branch adds im*eps to one component at a time: only that component's real part becomes x + 0.0.
    N = 2051
    cv = cyc_colors(N, 3)
    x_np = x_with_zeros(N, 15)
    x = torch.from_numpy(x_np).to(dev)
    log = []

    def f(dx, xx):
        log.append(np.array(xx.cpu().numpy(), copy=True))
        dx.copy_(xx * (1.0 + torch.atan2(torch.zeros_like(xx.real), xx.real)))

    def f_np(dx, xx):
        dx[:] = xx * (1.0 + np.arctan2(np.zeros_like(xx.real), xx.real))
    olog = []

    def f_np_rec(dx, xx):
        olog.append(np.array(xx, copy=True))
        f_np(dx, xx)
    if dense:
        n = 40                                                  # dense branch: n calls
        x = x[:n].contiguous()
        x_np = x_np[:n]
        J = pkg.zeros_colmajor(n, n, dev)
        pkg.finite_difference_jacobian_(J, f, x, pkg.JacobianCache(x, "complex"))
        ref = np.zeros(n * n)
        oracle.jacobian_complex(oracle.Problem.dense(n, n), ref, f_np_rec, x_np.copy())
        got = J.cpu().numpy().reshape(-1, order="F")
    else:
        colptr, rowval = tridiag_csc(N)
        J = pkg.SparseMatrixCSC(N, N, t64(colptr), t64(rowval), torch.full((len(rowval),), float("nan"), dtype=torch.float64,
                                                                             device=dev))
        pkg.finite_difference_jacobian_(J, f, x, pkg.JacobianCache(x, "complex", colorvec=cv, sparsity=J))
        ref = np.full(len(rowval), np.nan)
        oracle.jacobian_complex(oracle.Problem.csc_same(N, N, colptr, rowval), ref, f_np_rec, x_np.copy(), colorvec=cv)
        got = J.nzval.cpu().numpy()
    torch.cuda.synchronize()
    assert len(log) == len(olog)
    for i, (a, b) in enumerate(zip(log, olog)):
        assert_same_bits(a.view(np.float64), b.view(np.float64), f"argument of f! call {i}")
    assert_same_bits(got, ref, "J")
