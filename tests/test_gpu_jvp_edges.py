"""The device Jacobian-vector product (fdb_jvp, kernels_jvp.cuh; src/jvp.jl:238-274) at IEEE edges, step overrides, tile
boundary sizes, misaligned buffers, several tiles per block, reused plans and aliased caches.

Every parity assert is a bit compare (_util.assert_same_bits) against the C restatement oracle.jvp given the same f.  On
exact-dot inputs (_util.exact_dot_xv: dot(x, v) is exact in any summation order) the device eps is compared with the
oracle's own eps; where an IEEE edge makes the dot inexact, the device eps is fed to the oracle.  The one tolerance is
the exact-arithmetic bound on eps over general data (test_gpu_jvp_eps_within_exact_dot_bound).

f is _util.GatherF: gathers and separately rounded * + - on CUDA tensors, so its numpy twin gives the same bits, and
every point it is called with is recorded and compared, in order."""
import ctypes as C
import math
import re

import numpy as np
import pytest

from _util import GatherF, assert_same_bits, exact_dot_xv, fdb_env, traced

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

FD = {"forward": 0, "central": 1}
U = 2.0 ** -53
BIG = 1_000_003
RELSTEPS = [None, 0.0, 1e-3, -1e-3, -0.0, 1.0]
ABSSTEPS = [None, 0.0, -0.0, 1e-160, 5e-324]
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 1e300, -1e300]


@pytest.fixture(scope="module")
def pkg(oracle):
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


def _dev(a, off=0):
    """A CUDA copy of a whose first element sits `off` elements into its allocation (off = 1: 8-byte aligned only)."""
    buf = torch.zeros(a.size + off, dtype=torch.float64, device="cuda")
    buf[off:] = torch.from_numpy(np.ascontiguousarray(a))
    return buf[off:]


def _run(pkg, oracle, xh, vh, m, fdtype, *, f_in=False, own_eps=True, off=None, buffers=False, alias=False, cache=None,
         seed=0, **steps):
    """One device JVP of GatherF(m, n) and the oracle's run; assert bit parity of eps (own_eps: the oracle's own eps;
    otherwise the device eps is fed to it), of every point f sees, the call count, jvp and cache.x1, and that x and v
    are left unchanged (x is cache.x1 itself when alias).  Returns (eps, oracle result, cache)."""
    off = off or {}
    n = xh.size
    g = GatherF(m, n, seed)
    x, v = _dev(xh, off.get("x", 0)), _dev(vh, off.get("v", 0))
    fin_h = fin = None
    if f_in:
        fin_h = np.zeros(m)
        g.np_f([])(fin_h, xh.copy())
        fin = _dev(fin_h, off.get("f_in", 0))
    if cache is None:
        if alias:
            cache = pkg.JVPCache(x, _dev(np.zeros(m), off.get("fx1", 0)), fdtype)
        elif buffers or m != n:
            cache = pkg.JVPCache(_dev(np.full(n, np.nan), off.get("x1", 0)), _dev(np.full(m, np.nan), off.get("fx1", 0)),
                                 fdtype)
        else:
            cache = pkg.JVPCache(x, fdtype)
    jvp = _dev(np.full(m, np.nan), off.get("jvp", 0))
    dlog, olog = [], []
    pkg.finite_difference_jvp_(jvp, g.torch_f(dlog, x.device), x, v, cache, fin, **steps)
    torch.cuda.synchronize()
    eps = float(cache._last_plan.eps()[0])
    kw = dict(fdtype=FD[fdtype], f_in=fin_h, alias_x1=alias, **steps)
    r = oracle.jvp(g.np_f(olog), xh.copy(), vh.copy(), m, eps_override=None if own_eps else eps, **kw)
    what = f"{fdtype} n={n} m={m} {steps}"
    assert_same_bits(np.array([eps]), np.array([r["eps"]]), f"{what}: eps")
    assert len(dlog) == len(olog) == r["fcalls"] == (1 if f_in and fdtype == "forward" else 2), what
    for i, (a, b) in enumerate(zip(dlog, olog)):
        assert_same_bits(a, b, f"{what}: argument of f call {i}")
    assert_same_bits(jvp, r["jvp"], f"{what}: jvp")
    assert_same_bits(cache.x1, r["x1"][:n], f"{what}: cache.x1")
    if alias:
        assert cache.x1 is x
    else:
        assert_same_bits(x, xh, f"{what}: caller's x modified")
    assert_same_bits(v, vh, f"{what}: v modified")
    return eps, r, cache


def _sizes():
    out = []
    for n in (0, 1, 2, 1023, 1024, 1025, 2047, 2048, 2049, BIG):
        for m in sorted({k for k in (0, 1, n - 1, n, n + 1, 3 * n) if k >= 0}):
            out.append((n, m))
    return out


# ------------------------------------------------------------------------------------------------ sizes, m != n
@pytest.mark.parametrize("mode", ["forward", "forward_fin", "central"])
@pytest.mark.parametrize("n,m", _sizes())
def test_gpu_jvp_sizes(pkg, oracle, n, m, mode):
    xh, vh = exact_dot_xv(n, n + 3 * m, "neg" if n % 2 else "unit")
    _run(pkg, oracle, xh, vh, m, "central" if mode == "central" else "forward", f_in=mode == "forward_fin", seed=n)


@pytest.mark.parametrize("fdtype", list(FD))
@pytest.mark.parametrize("kind", ["unit", "big", "tiny", "neg", "zero"])
@pytest.mark.parametrize("n", [2049, BIG - 1])
def test_gpu_jvp_exact_dot_kinds(pkg, oracle, n, kind, fdtype):
    xh, vh = exact_dot_xv(n, 31, kind)
    eps, r, _ = _run(pkg, oracle, xh, vh, n, fdtype)
    if kind == "zero":                                   # sqrt(0) = 0: eps = absstep = relstep
        assert eps == oracle.default_relstep(FD[fdtype])


# ------------------------------------------------------------------------------------------------ step overrides, dir
@pytest.mark.parametrize("absstep", ABSSTEPS)
@pytest.mark.parametrize("relstep", RELSTEPS)
@pytest.mark.parametrize("fdtype,dir", [("forward", 1.0), ("forward", -1.0), ("forward", 0.3), ("central", 1.0),
                                        ("central", -1.0), ("central", 0.3)])
def test_gpu_jvp_step_overrides(pkg, oracle, fdtype, dir, relstep, absstep):
    for kind in ("unit", "neg"):
        xh, vh = exact_dot_xv(2049, 5, kind)
        _run(pkg, oracle, xh, vh, 2049, fdtype, relstep=relstep, absstep=absstep, dir=dir)


# ------------------------------------------------------------------------------------------------ IEEE edges
@pytest.mark.parametrize("fdtype", list(FD))
@pytest.mark.parametrize("which", ["x", "v"])
@pytest.mark.parametrize("edge", EDGES)
def test_gpu_jvp_edges(pkg, oracle, edge, which, fdtype):
    n = 3001
    xh, vh = exact_dot_xv(n, 12, "unit")
    for i in (0, 1, 1023, 1024, 1025, 2047, 2048, n - 1):
        (xh if which == "x" else vh)[i] = edge
    exact = bool(np.isnan(edge) or np.isinf(edge) or edge == 0.0)       # the dot stays order-independent
    _run(pkg, oracle, xh, vh, n, fdtype, own_eps=exact)


@pytest.mark.parametrize("fdtype", list(FD))
def test_gpu_jvp_zero_and_nan_v(pkg, oracle, fdtype):
    n = 2049
    xh, _ = exact_dot_xv(n, 13, "unit")
    vz = np.where(np.arange(n) % 3 == 0, -0.0, 0.0)
    eps, _, _ = _run(pkg, oracle, xh, vz, n, fdtype, relstep=1e-3, absstep=2.0 ** -30)
    assert eps == 2.0 ** -30
    eps, r, _ = _run(pkg, oracle, xh, np.full(n, np.nan), n, fdtype)
    assert math.isnan(eps) and np.isnan(r["jvp"]).all()


# ------------------------------------------------------------------------------------------------ misaligned buffers
@pytest.mark.parametrize("target,fdtype", [(t, fd) for t in ("x", "v", "x1", "fx1", "jvp", "f_in", "all") for fd in FD
                                           if (t, fd) != ("f_in", "central")])          # central never reads f_in
def test_gpu_jvp_misaligned(pkg, oracle, target, fdtype):
    # x or v shifted by one element sends the dot and both point passes through their element loops (al_xv = 0); x1
    # alone, only the point passes (al_x1 = 0).  n is odd, so the dot's last pair is a lone j.
    names = ("x", "v", "x1", "fx1", "jvp", "f_in")
    off = {k: 1 for k in names} if target == "all" else {target: 1}
    xh, vh = exact_dot_xv(BIG, 17, "neg")
    _run(pkg, oracle, xh, vh, BIG, fdtype, f_in=fdtype == "forward" and target in ("f_in", "all"), off=off, buffers=True)


# ------------------------------------------------------------------------------------------------ several tiles per block
@pytest.mark.parametrize("fdtype", list(FD))
@pytest.mark.parametrize("sm", [1, 3])
def test_gpu_jvp_multiwave(pkg, oracle, sm, fdtype):
    tiles = (BIG + 1023) // 1024
    xh, vh = exact_dot_xv(BIG, 19, "neg")
    with fdb_env(SM_COUNT=sm):
        kern = traced(lambda: _run(pkg, oracle, xh, vh, BIG, fdtype, buffers=True, off={"v": int(sm == 3)}))
    for name, count in (("jvp_dot_eps", 1), ("jvp_point", 1 if fdtype == "forward" else 2)):
        ks = [k for k in kern if re.search(r"\b" + name + r"\b", k[0])]
        assert len(ks) == count, (name, [k[0][:50] for k in kern])
        for k in ks:
            assert tiles / k[1] >= 3, f"{name}: grid {k[1]} gives {tiles / k[1]:.1f} tiles per block"


# ------------------------------------------------------------------------------------------------ one plan, many calls
@pytest.mark.parametrize("fdtype", list(FD))
def test_gpu_jvp_reused_plan(pkg, oracle, fdtype):
    # A Newton-Krylov solver calls the JVP once per iteration on one cache with x and v rewritten in place: each call's
    # eps must come from that call's x, v and steps (the dot's last-block ticket is reset for the next call).
    n, m = 5001, 5002
    g = GatherF(m, n, 3)
    x, v = _dev(np.zeros(n)), _dev(np.zeros(n))
    cache = pkg.JVPCache(_dev(np.zeros(n)), _dev(np.zeros(m)), fdtype)
    jvp = _dev(np.zeros(m))
    fin = _dev(np.zeros(m))
    calls = [dict(seed=1, kind="unit"),
             dict(seed=1, kind="unit"),                                  # repeated: the same bits
             dict(seed=2, kind="neg"),                                   # x and v rewritten
             dict(seed=2, kind="neg", vseed=3),                          # v alone rewritten
             dict(seed=2, kind="neg", vseed=3, relstep=1e-3),
             dict(seed=2, kind="neg", vseed=3, relstep=1e-3, absstep=1e3),
             dict(seed=2, kind="neg", vseed=3, dir=-1.0),
             dict(seed=4, kind="unit", f_in=True),
             dict(seed=4, kind="unit"),                                  # f_in omitted again
             dict(seed=5, kind="big", f_in=True, relstep=2.0 ** -20, dir=0.3)]
    prev = None
    for k, c in enumerate(calls):
        xh, vh = exact_dot_xv(n, c["seed"], c["kind"])
        if "vseed" in c:
            vh = exact_dot_xv(n, c["vseed"], c["kind"])[1]
        x.copy_(torch.from_numpy(xh))
        v.copy_(torch.from_numpy(vh))
        steps = {s: c[s] for s in ("relstep", "absstep", "dir") if s in c}
        fin_h = None
        if c.get("f_in"):
            fin_h = np.zeros(m)
            g.np_f([])(fin_h, xh)
            fin.copy_(torch.from_numpy(fin_h))
        dlog, olog = [], []
        pkg.finite_difference_jvp_(jvp, g.torch_f(dlog, x.device), x, v, cache, fin if c.get("f_in") else None, **steps)
        torch.cuda.synchronize()
        eps = float(cache._last_plan.eps()[0])
        r = oracle.jvp(g.np_f(olog), xh, vh, m, fdtype=FD[fdtype], f_in=fin_h, **steps)
        assert_same_bits(np.array([eps]), np.array([r["eps"]]), f"call {k} {c}: eps")
        assert len(dlog) == r["fcalls"], f"call {k}"
        for a, b in zip(dlog, olog):
            assert_same_bits(a, b, f"call {k}: points")
        assert_same_bits(jvp, r["jvp"], f"call {k}: jvp")
        if k == 1:
            assert_same_bits(jvp, prev, "a repeated call")
        prev = jvp.clone()
    assert cache._last_plan.counters()["jacobians"] == len(calls)


# ------------------------------------------------------------------------------------------------ aliasing
@pytest.mark.parametrize("fdtype", list(FD))
@pytest.mark.parametrize("n", [1025, BIG])
def test_gpu_jvp_aliased_cache(pkg, oracle, n, fdtype):
    # JVPCache(x, fx1) keeps x1 = the caller's x, as jvp.jl:73-80 does: central evaluates f at (x - eps v) + eps v and
    # leaves x there; the point kernel reads and writes x in place
    xh, vh = exact_dot_xv(n, 23, "unit")
    _run(pkg, oracle, xh, vh, n, fdtype, alias=True)


@pytest.mark.parametrize("mode", ["forward_fin", "central"])
def test_gpu_jvp_cacheless(pkg, oracle, mode):
    # finite_difference_jvp!(jvp, f, x, v, fdtype, f_in) (jvp.jl:205-223).  The reference's JVPCache(x, f_in) aliases
    # x1 to x and moves the caller's x; the mirror copies x, so x is unchanged and jvp is the reference's
    n = 4099
    xh, vh = exact_dot_xv(n, 29, "neg")
    g = GatherF(n, n, 1)
    x, v = _dev(xh), _dev(vh)
    jvp = _dev(np.full(n, np.nan))
    fin_h = None
    dlog, olog = [], []
    if mode == "forward_fin":
        fin_h = np.zeros(n)
        g.np_f([])(fin_h, xh)
        pkg.finite_difference_jvp_(jvp, g.torch_f(dlog, x.device), x, v, None, _dev(fin_h))
    else:
        pkg.finite_difference_jvp_(jvp, g.torch_f(dlog, x.device), x, v, "central")
    torch.cuda.synchronize()
    r = oracle.jvp(g.np_f(olog), xh, vh, n, fdtype=1 if mode == "central" else 0, f_in=fin_h)
    assert_same_bits(x, xh, "caller's x")
    assert len(dlog) == r["fcalls"]
    for a, b in zip(dlog, olog):
        assert_same_bits(a, b, "points")
    assert_same_bits(jvp, r["jvp"], "jvp")


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.mark.parametrize("fdtype", list(FD))
def test_gpu_jvp_abi_plan_scratch(pkg, oracle, fdtype):
    # fdb_jvp with d_x1 = d_fx1 = NULL works in the plan's own scratch: the same bits as caller buffers
    L = pkg._lib
    n = 4099
    xh, vh = exact_dot_xv(n, 37, "unit")
    x, v = _dev(xh), _dev(vh)
    plan = pkg.JVPCache(x, fdtype).plan(n, n)
    addr = C.cast(L.synth().fdbs_tridiag, C.c_void_p).value
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    fin = _dev(np.zeros(n))
    out = []
    for use_buffers in (False, True, False):
        for f_in in ((None, fin) if fdtype == "forward" else (None,)):
            ctx = L.TridiagCtx(n, 0)
            jvp = _dev(np.full(n, np.nan))
            x1, fx1 = _dev(np.zeros(n)), _dev(np.zeros(n))
            if f_in is not None:
                assert L.synth().fdbs_tridiag(C.cast(C.pointer(ctx), C.c_void_p), fin.data_ptr(), x.data_ptr(), 1,
                                              n + 1, n + 1, stream) == 0                     # f_in = f(x)
            L.check(L.lib().fdb_jvp(plan.handle, addr, C.cast(C.pointer(ctx), C.c_void_p), jvp.data_ptr(), x.data_ptr(),
                                    v.data_ptr(), x1.data_ptr() if use_buffers else None,
                                    fx1.data_ptr() if use_buffers else None, None if f_in is None else f_in.data_ptr(),
                                    L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, stream))
            torch.cuda.synchronize()
            fin_h = None if f_in is None else f_in.cpu().numpy()
            r = oracle.jvp(oracle.native_fn("synth_tridiag"), xh, vh, n, fdtype=FD[fdtype], f_in=fin_h,
                           ctx=oracle.SynthTridiagCtx(n, 1))
            assert_same_bits(np.array([plan.eps()[0]]), np.array([r["eps"]]), "eps")
            assert_same_bits(jvp, r["jvp"], f"jvp buffers={use_buffers} f_in={f_in is not None}")
            if use_buffers:
                assert_same_bits(x1, r["x1"][:n], "x1")
            out.append(jvp.cpu().numpy())
    assert_same_bits(out[0], out[-1])


# ------------------------------------------------------------------------------------------------ exact-arithmetic bound
def _two_prod(a, b):
    """Dekker's error-free product (no FMA): a*b = p + e exactly, for moderate magnitudes."""
    def split(t):
        c = 134217729.0 * t
        hi = c - (c - t)
        return hi, t - hi
    p = a * b
    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


@pytest.mark.parametrize("case", ["positive", "negative", "cancelling", "mixed"])
@pytest.mark.parametrize("n", [4099, BIG])
def test_gpu_jvp_eps_within_exact_dot_bound(pkg, oracle, n, case):
    # General data: the device's tree order rounds differently from any CPU loop, so eps is held to the exact dot d:
    # |d_hat - d| <= B = gamma_n * sum |x_j v_j| in any summation order, so eps = relstep * sqrt(|d_hat|) lies in
    # [relstep * sqrt(max(|d| - B, 0)), relstep * sqrt(|d| + B)] * (1 +- 4u).  A dropped or doubled tile, or a missing
    # fabs, leaves it.  (absstep = 0: eps is the relative branch whenever d_hat != 0.)
    rng = np.random.default_rng(n + len(case))
    x = rng.uniform(0.5, 2.0, n) * 10.0 ** rng.integers(-3, 3, n)
    v = rng.uniform(0.5, 2.0, n)
    if case == "negative":
        v = -v
    elif case == "mixed":
        v = v * np.where(rng.random(n) < 0.45, -1.0, 1.0)
    elif case == "cancelling":                       # x.v ~ 0 with |x_j v_j| ~ 1
        x = rng.uniform(0.5, 2.0, n)
        v = 1.0 / x
        v[1::2] = -(x[0:n - 1:2] * v[0:n - 1:2]) / x[1::2]
        v[-1] = 1e-8 / x[-1]                         # n is odd: the unpaired last product is small too
    p, e = _two_prod(x, v)
    d = math.fsum(np.concatenate([p, e]))
    S = math.fsum(np.abs(p)) * (1 + 4 * U)
    B = n * U / (1 - n * U) * S
    rel = math.sqrt(np.finfo(float).eps)
    xs, vs = _dev(x), _dev(v)
    L = pkg._lib
    for fdtype in ("forward", "central"):
        cache = pkg.JVPCache(xs, fdtype)
        jvp = _dev(np.zeros(n))
        rs = rel if fdtype == "forward" else float(np.cbrt(np.finfo(float).eps))
        ctx = L.TridiagCtx(n, 0)
        f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
        pkg.finite_difference_jvp_(jvp, f, xs, vs, cache, relstep=rs, absstep=0.0)
        torch.cuda.synchronize()
        eps = float(cache._last_plan.eps()[0])
        lo = rs * math.sqrt(max(abs(d) - B, 0.0)) * (1 - 4 * U)
        hi = rs * math.sqrt(abs(d) + B) * (1 + 4 * U)
        assert lo <= eps <= hi, f"{case} {fdtype}: eps {eps!r} outside [{lo!r}, {hi!r}] (d = {d!r}, B = {B!r})"
        if case != "cancelling":
            assert (hi - lo) < 1e-6 * hi                 # the bound is tight enough to see one tile of 1024 terms
        r = oracle.jvp(oracle.native_fn("synth_tridiag"), x, v, n, fdtype=FD[fdtype], relstep=rs, absstep=0.0,
                       eps_override=eps, ctx=oracle.SynthTridiagCtx(n, 1))
        assert_same_bits(jvp, r["jvp"], f"{case} {fdtype}: jvp at the device eps")


# ------------------------------------------------------------------------------------------------ rejected buffers
def _reject_cases(n, m):
    z = lambda k, **kw: torch.zeros(k, device="cuda", dtype=torch.float64, **kw)     # noqa: E731
    base = z(2 * m)
    return [
        ("strided fx1", dict(fx1=base[::2]), ValueError, base),
        ("strided x1", dict(x1=z(2 * n)[::2]), ValueError, None),
        ("float32 x1", dict(x1=torch.zeros(n, device="cuda", dtype=torch.float32)), TypeError, None),
        ("float32 fx1", dict(fx1=torch.zeros(m, device="cuda", dtype=torch.float32)), TypeError, None),
        ("short x1", dict(x1=z(n - 1)), ValueError, None),
        ("short fx1", dict(fx1=z(m - 1)), ValueError, None),
        ("long fx1", dict(fx1=z(m + 1)), ValueError, None),
        ("CPU f_in", dict(f_in=torch.zeros(m, dtype=torch.float64)), TypeError, None),
        ("strided f_in", dict(f_in=z(2 * m)[::2]), ValueError, None),
        ("float32 f_in", dict(f_in=torch.zeros(m, device="cuda", dtype=torch.float32)), TypeError, None),
        ("short f_in", dict(f_in=z(m - 1)), ValueError, None),
    ]


@pytest.mark.parametrize("case", range(11))
def test_gpu_jvp_rejects_bad_buffers(pkg, case):
    # The device reads and writes n / m contiguous doubles from each buffer: the mirror rejects what would be read past
    # its end or written outside the caller's view, before anything runs.  A strided fx1 = base[::2] would otherwise have
    # m doubles written from its first element, over base's odd elements.
    n, m = 300, 301
    what, bad, exc, watch = _reject_cases(n, m)[case]
    x, v = _dev(exact_dot_xv(n, 1, "unit")[0]), _dev(exact_dot_xv(n, 1, "unit")[1])
    x1 = bad.get("x1", torch.zeros(n, dtype=torch.float64, device="cuda"))
    fx1 = bad.get("fx1", torch.zeros(m, dtype=torch.float64, device="cuda"))
    cache = pkg.JVPCache(x1, fx1, "forward")
    jvp = _dev(np.full(m, np.nan))
    calls = []
    with pytest.raises(exc):
        pkg.finite_difference_jvp_(jvp, lambda fx, xx: calls.append(1), x, v, cache, bad.get("f_in"))
    torch.cuda.synchronize()
    assert not calls, what
    assert torch.isnan(jvp).all(), what
    if watch is not None:
        assert_same_bits(watch, np.zeros(watch.numel()), f"{what}: memory outside the view written")
    if "f_in" in bad:                             # central mode never reads f_in (jvp.jl:264-269)
        pkg.finite_difference_jvp_(jvp, lambda fx, xx: fx.copy_(xx[:1].expand(m)), x, v, pkg.JVPCache(x1, fx1, "central"),
                                   bad["f_in"])


def test_gpu_jvp_empty_f_in_is_given(pkg, oracle):
    # m = 0 with f_in: f_in has no storage, but it is given, so f(fx1, x) is not evaluated (one f call, as jvp.jl:257-258)
    xh, vh = exact_dot_xv(5, 2, "unit")
    _run(pkg, oracle, xh, vh, 0, "forward", f_in=True)
