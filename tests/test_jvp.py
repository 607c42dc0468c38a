"""Jacobian-vector product (SURVEY.md §8f rank 2; src/jvp.jl:238-274): oracle pinned on the reference tests' JVP
fixtures (test/finitedifftests.jl:419-478), CUDA path bit-compared with the oracle."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits


def _iipf(fvec, x):
    fvec[0] = (x[0] + 3) * (x[1] ** 3 - 7) + 18
    fvec[1] = np.sin(x[1] * np.exp(x[0]) - 1)


def _J_ref(x):
    return np.array([[-7 + x[1] ** 3, 3 * (3 + x[0]) * x[1] ** 2],
                     [np.exp(x[0]) * x[1] * np.cos(1 - np.exp(x[0]) * x[1]), np.exp(x[0]) * np.cos(1 - np.exp(x[0]) * x[1])]])


def test_oracle_jvp_kats(oracle, golden):
    # finitedifftests.jl:470-478: forward < 1e-6, dir=-1, relstep, f_in, central < 1e-8; jvp_ref = J_ref * vdir (:426)
    x = np.array(golden["analytic2x2"]["x"])
    v = np.random.default_rng(4).random(2)
    ref = _J_ref(x) @ v
    err = lambda a: float(np.max(np.abs(a - ref)))
    r = oracle.jvp(_iipf, x, v, 2)
    assert err(r["jvp"]) < 1e-6 and r["fcalls"] == 2
    assert err(oracle.jvp(_iipf, x, v, 2, fdtype=1)["jvp"]) < 1e-8
    assert err(oracle.jvp(_iipf, x, v, 2, relstep=float(np.sqrt(np.finfo(float).eps)))["jvp"]) < 1e-6
    y = np.zeros(2)
    _iipf(y, x)
    r = oracle.jvp(_iipf, x, v, 2, f_in=y)
    assert err(r["jvp"]) < 1e-6 and r["fcalls"] == 1

    def iipff(df, xx):                      # finitedifftests.jl:409: errors if any component is perturbed upwards
        if not np.all(xx <= x):
            raise AssertionError("perturbed upward")
        _iipf(df, xx)

    assert err(oracle.jvp(iipff, x, v, 2, dir=-1.0)["jvp"]) < 1e-6
    # central calls f(fx1, x - eps v) BEFORE f(jvp, x + eps v)  (jvp.jl:264-267)
    log = []

    def rec(df, xx):
        log.append(xx.copy())
        _iipf(df, xx)

    r = oracle.jvp(rec, x, v, 2, fdtype=1)
    assert len(log) == 2 and np.all(log[0] < x) and np.all(log[1] > x)
    np.testing.assert_allclose(log[1] - x, r["eps"] * v, rtol=1e-6)
    # eps = max(relstep*sqrt(|x.v|), absstep)
    rel = np.sqrt(np.finfo(float).eps)
    assert oracle.jvp(_iipf, x, v, 2)["eps"] == pytest.approx(max(rel * np.sqrt(abs(x @ v)), rel), rel=1e-15)


torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.mark.gpu
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_gpu_jvp_bitexact(pkg, oracle, fdtype):
    dev = torch.device("cuda:0")
    L = pkg._lib
    for N in (1_000_003, 4099, 2, 1):
        x = torch.empty(N, dtype=torch.float64, device=dev)
        v = torch.empty(N, dtype=torch.float64, device=dev)
        L.synth().fdbs_fill_x(x.data_ptr(), N, 101, None)
        L.synth().fdbs_fill_x(v.data_ptr(), N, 202, None)
        jvp = torch.full((N,), float("nan"), dtype=torch.float64, device=dev)
        ctx = L.TridiagCtx(N, 0)
        if N % 2 == 1 and N > 1:
            pass
        f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
        cache = pkg.JVPCache(x, fdtype)
        xb, vb = x.clone(), v.clone()
        pkg.finite_difference_jvp_(jvp, f, x, v, cache)
        torch.cuda.synchronize()
        assert_same_bits(x, xb, allow_nan=False)
        assert_same_bits(v, vb, allow_nan=False)
        eps = cache._last_plan.eps()[0]
        xh, vh = oracle.fill_x(N, 101), oracle.fill_x(N, 202)
        own = oracle.jvp(oracle.native_fn("synth_tridiag"), xh, vh, N, fdtype=0 if fdtype == "forward" else 1,
                         ctx=oracle.SynthTridiagCtx(N, 1))
        assert eps == pytest.approx(own["eps"], rel=1e-13)
        r = oracle.jvp(oracle.native_fn("synth_tridiag"), xh, vh, N, fdtype=0 if fdtype == "forward" else 1, eps_override=eps,
                       ctx=oracle.SynthTridiagCtx(N, 1))
        assert ctx.calls == r["fcalls"] == 2
        assert_same_bits(jvp.cpu().numpy(), r["jvp"], allow_nan=False)
        assert_same_bits(cache.x1.cpu().numpy(), r["x1"], allow_nan=False)                         # cache.x1 ends as x + eps*v (jvp.jl:260/:266)
        # linear f: J*v exactly the stencil applied to v (up to cancellation)
        Jv = np.zeros(N)
        import _util
        _util.f_tridiag(Jv, vh) if N > 1 else Jv.__setitem__(0, -2 * vh[0])
        np.testing.assert_allclose(jvp.cpu().numpy(), Jv, atol=1e-6 if fdtype == "forward" else 1e-8)


@pytest.mark.gpu
def test_gpu_jvp_kats_python_callbacks(pkg, golden):
    # finitedifftests.jl:470-478 through the mirror
    dev = torch.device("cuda:0")
    xh = np.array(golden["analytic2x2"]["x"])
    vh = np.random.default_rng(4).random(2)
    x = torch.tensor(xh, dtype=torch.float64, device=dev)
    v = torch.tensor(vh, dtype=torch.float64, device=dev)
    ref = _J_ref(xh) @ vh

    def iipf(fvec, xx):
        fvec[0] = (xx[0] + 3) * (xx[1] ** 3 - 7) + 18
        fvec[1] = torch.sin(xx[1] * torch.exp(xx[0]) - 1)

    err = lambda t: float(np.max(np.abs(t.cpu().numpy() - ref)))
    jvp = torch.zeros(2, dtype=torch.float64, device=dev)
    fwd, cen = pkg.JVPCache(x, "forward"), pkg.JVPCache(x, "central")
    pkg.finite_difference_jvp_(jvp, iipf, x, v, fwd)
    assert err(jvp) < 1e-6
    pkg.finite_difference_jvp_(jvp, iipf, x, v, cen)
    assert err(jvp) < 1e-8
    pkg.finite_difference_jvp_(jvp, iipf, x, v, "central")                 # cache-less, Val{:central}
    assert err(jvp) < 1e-8
    pkg.finite_difference_jvp_(jvp, iipf, x, v, fwd, relstep=float(np.sqrt(np.finfo(float).eps)))
    assert err(jvp) < 1e-6
    y = torch.zeros(2, dtype=torch.float64, device=dev)
    iipf(y, x)
    calls = []

    def counted(fvec, xx):
        calls.append(1)
        iipf(fvec, xx)

    pkg.finite_difference_jvp_(jvp, counted, x, v, fwd, y)
    assert err(jvp) < 1e-6 and len(calls) == 1

    def iipff(df, xx):
        if not bool(torch.all(xx <= x)):
            raise RuntimeError("perturbed upward")
        iipf(df, xx)

    pkg.finite_difference_jvp_(jvp, iipff, x, v, fwd, dir=-1)
    assert err(jvp) < 1e-6
    with pytest.raises(RuntimeError, match="perturbed upward"):
        pkg.finite_difference_jvp_(jvp, iipff, x, v, fwd)
    with pytest.raises(ValueError, match="complex"):                       # jvp.jl:248-250
        pkg.finite_difference_jvp_(jvp, iipf, x, v, pkg.JVPCache(x, "complex"))
