"""Gradients of a scalar f (src/gradients.jl:390-473).

CPU: the C restatement (scalar_oracle/, written separately from the Jacobian oracle) against the reference's gradient
tests (test/finitedifftests.jl:173-202) and, bit for bit, against a line-by-line Python transcription.
GPU: finite_difference_gradient! runs the dense Jacobian plan with m = 1; bit-compared with the gradient restatement —
so the claim "the gradient is the dense column branch with m = 1" is tested, not assumed."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, gradient_transcribed
from scalar_oracle import fd_scalar_oracle as so

f64 = np.float64
EPS = np.finfo(float).eps


@pytest.fixture(scope="module")
def soracle():
    so.build()
    so.lib()
    return so


def err_func(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))))


def test_kat_gradients(soracle):
    # finitedifftests.jl:173-202: f(x) = 2x[1] + x[2]^2
    x = np.random.default_rng(3).random(2)
    z = x.copy()
    f = lambda v: 2 * v[0] + v[1] ** 2
    fc = lambda v: 2 * v[0] + v[1] * v[1]          # complex-step twin (x[2]^2 of a complex number)

    def ff(k):                                      # errors when a component is perturbed upwards
        if not np.all(k <= z):
            raise AssertionError("perturbed upward")
        return f(k)

    df_ref = np.array([2.0, 2 * x[1]])
    assert err_func(soracle.gradient(f, x, so.FORWARD)["df"], df_ref) < 1e-4
    assert err_func(soracle.gradient(ff, x, so.FORWARD, dir=-1.0)["df"], df_ref) < 1e-4
    assert err_func(soracle.gradient(f, x, so.FORWARD, relstep=np.sqrt(EPS))["df"], df_ref) < 1e-4
    assert err_func(soracle.gradient(f, x, so.CENTRAL)["df"], df_ref) < 1e-8
    assert err_func(soracle.gradient(fc, x, so.COMPLEX)["df"], df_ref) < 1e-15
    r = soracle.gradient(f, x, so.FORWARD, fx=f(x))
    assert err_func(r["df"], df_ref) < 1e-4 and r["fcalls"] == 2
    assert soracle.gradient(f, x, so.FORWARD)["fcalls"] == 3
    assert soracle.gradient(f, x, so.CENTRAL)["fcalls"] == 4


def test_kat_gradient_of_sum_is_ones(soracle):
    # finitedifftests.jl:586-590 (the gradient side of the thread-safety block): gradient of sum is ones
    for fd in (so.FORWARD, so.CENTRAL):
        np.testing.assert_allclose(soracle.gradient(lambda v: float(np.sum(v)), np.ones(2), fd)["df"], np.ones(2))
    np.testing.assert_allclose(soracle.gradient(lambda v: complex(np.sum(v)), np.ones(2), so.COMPLEX)["df"], np.ones(2))


EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, 5e-324, 1e300, -1e300, 1.0]


def _poly(v):
    with np.errstate(all="ignore"):
        s = f64(0)
        for k in range(len(v)):
            s = s + f64(0.5) * v[k] * v[k] * v[k] + v[k] * v[(k + 1) % len(v)]
        return s


def test_oracle_matches_transcription_random(soracle):
    rng = np.random.default_rng(390)
    for trial in range(300):
        n = int(rng.integers(0, 7))
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
        for k in range(n):
            if rng.random() < 0.3:
                x[k] = EDGES[rng.integers(len(EDGES))]
        fd = int(rng.integers(0, 2))
        relstep = [None, 0.0, 1e-3][rng.integers(3)]
        absstep = [None, 0.0, 1e-6, 1e-320][rng.integers(4)]
        dir = [1.0, -1.0][rng.integers(2)]
        fx = [None, 0.25][rng.integers(2)] if fd == 0 else None
        df, pts = gradient_transcribed(_poly, x, fd, fx, relstep, absstep, dir)
        r = soracle.gradient(_poly, x, fd, fx=fx, relstep=relstep, absstep=absstep, dir=dir, log=True)
        assert r["fcalls"] == len(pts)
        for p, q in zip(r["points"], pts):
            assert_same_bits(p, q, f"trial {trial}: point")
        assert_same_bits(r["df"], df, f"trial {trial}: df")


# ------------------------------------------------------------------------------------------------ GPU
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


def _problem(pkg, n, complex_=False):
    rng = np.random.default_rng(11 + n)
    a, w = 0.5 + rng.random(n), rng.random(n) * 2 - 1
    d_a, d_w = torch.from_numpy(a).cuda(), torch.from_numpy(w).cuda()
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0xBEEF + n, None)
    ctx = pkg._lib.ScalarCtx(n, d_a.data_ptr(), d_w.data_ptr(), 0)
    name = "fdbs_quartic_c" if complex_ else "fdbs_quartic"
    fn = pkg.NativeFn(C.cast(getattr(pkg._lib.synth(), name), C.c_void_p).value, ctx, keepalive=(d_a, d_w))
    return x, fn, ctx, so.SynthScalar(n, a, w)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 1000, 20000])
@pytest.mark.parametrize("mode", ["forward", "forward_fx", "central", "complex", "forward_dir"])
def test_gpu_gradient_bitexact(pkg, n, mode):
    x, fn, ctx, twin = _problem(pkg, n, complex_=mode == "complex")
    xh = x.cpu().numpy().copy()
    fd = {"forward": "forward", "forward_fx": "forward", "forward_dir": "forward", "central": "central",
          "complex": "complex"}[mode]
    dir = -1.0 if mode == "forward_dir" else 1.0
    fx = twin(xh) if mode == "forward_fx" else None
    if fx is None:
        cache = pkg.GradientCache(torch.zeros(n, dtype=torch.float64, device="cuda"), x, fd, max_batch=64)
    else:
        cache = pkg.GradientCache(fx, None, None, torch.zeros_like(x), fd, max_batch=64)
    df = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
    pkg.finite_difference_gradient_(df, fn, x, cache, dir=dir)
    torch.cuda.synchronize()
    assert_same_bits(x.cpu().numpy(), xh, "x modified", allow_nan=False)
    if mode == "complex":
        ref = so.gradient(twin.native("synth_quartic_c"), xh, so.COMPLEX)
    else:
        ref = so.gradient(twin.native("synth_quartic"), xh, so.FORWARD if fd == "forward" else so.CENTRAL, fx=fx, dir=dir)
    assert_same_bits(df.cpu().numpy(), ref["df"], f"{mode} n={n}", allow_nan=False)
    assert ctx.calls == ref["fcalls"]
    assert cache._last_plan.counters()["f_invocations"] > (1 if n > 64 else 0)


@pytest.mark.gpu
def test_gpu_gradient_python_f_and_errors(pkg):
    x = torch.rand(2, dtype=torch.float64, device="cuda")
    df_ref = torch.stack([torch.tensor(2.0, dtype=torch.float64, device="cuda"), 2 * x[1]])
    f = lambda v: 2 * v[0] + v[1] ** 2
    for fd, tol in (("forward", 1e-4), ("central", 1e-8)):
        assert float((pkg.finite_difference_gradient(f, x, fd) - df_ref).abs().max()) < tol
    with pytest.raises(TypeError):
        pkg.finite_difference_gradient(f, x.to(torch.complex128), "forward")
    with pytest.raises(TypeError):
        pkg.finite_difference_gradient(f, 1.0, "forward")
    with pytest.raises(TypeError):
        pkg.finite_difference_gradient(f, x.cpu(), "forward")

    class Boom(Exception):
        pass

    def g(v):
        raise Boom()

    with pytest.raises(Boom):
        pkg.finite_difference_gradient(g, x, "central")


@pytest.mark.gpu
def test_gpu_gradient_n1e5_forward(pkg, soracle):
    # n = 10^5 with 25 batches of 4096 points: bit-identical to the restatement (fdbs_sumsq and its CPU twin)
    n = 100_000
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0xF00D, None)
    ctx = pkg._lib.ScalarCtx(n, None, None, 0)
    fn = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_sumsq, C.c_void_p).value, ctx)
    cache = pkg.GradientCache(torch.zeros(n, dtype=torch.float64, device="cuda"), x, "forward", max_batch=4096)
    df = pkg.finite_difference_gradient(fn, x, cache)
    torch.cuda.synchronize()
    xh = x.cpu().numpy().copy()
    ref = soracle.gradient(soracle.SynthScalar(n).native("synth_sumsq"), xh, so.FORWARD)
    assert_same_bits(df.cpu().numpy(), ref["df"], "n=1e5 forward", allow_nan=False)
    assert ctx.calls == ref["fcalls"] == n + 1
    assert cache._last_plan.counters()["f_invocations"] == 1 + 25


@pytest.mark.gpu
def test_gpu_gradient_python_number_f(pkg, soracle):
    # f returning plain Python numbers (a Julia-style f returns a native Float64): stored as float64 / complex128
    xh = np.random.default_rng(5).random(2)
    x = torch.from_numpy(xh).cuda()
    df_ref = np.array([2.0, 2 * xh[1]])
    f_dev = lambda v: float(2 * v[0] + v[1] * v[1])
    f_host = lambda v: 2 * v[0] + v[1] * v[1]
    for fd, code, tol in (("forward", so.FORWARD, 1e-4), ("central", so.CENTRAL, 1e-8)):
        got = pkg.finite_difference_gradient(f_dev, x, fd).cpu().numpy()
        assert_same_bits(got, soracle.gradient(f_host, xh, code)["df"], f"{fd}, Python float f", allow_nan=False)
        assert err_func(got, df_ref) < tol
    got = pkg.finite_difference_gradient(lambda v: complex(2 * v[0] + v[1] * v[1]), x, "complex").cpu().numpy()
    assert err_func(got, df_ref) < 1e-15                      # finitedifftests.jl:184, Python complex f


@pytest.mark.gpu
def test_gpu_gradient_graph_replay_with_fx(pkg, soracle):
    # a numeric cache.fx is staged in one device slot kept on the cache: replays see the same arguments
    n = 1000
    x, fn, ctx, twin = _problem(pkg, n)
    xh = x.cpu().numpy().copy()
    fx = twin(xh)
    cache = pkg.GradientCache(fx, None, None, torch.zeros_like(x), "forward", max_batch=64, use_graph=True)
    df = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
    slots = set()
    for _ in range(3):
        pkg.finite_difference_gradient_(df, fn, x, cache)
        slots.add(cache._fin.data_ptr())
    torch.cuda.synchronize()
    ref = soracle.gradient(twin.native("synth_quartic"), xh, so.FORWARD, fx=fx)
    assert_same_bits(df.cpu().numpy(), ref["df"], "graph replay", allow_nan=False)
    assert len(slots) == 1
    c = cache._last_plan.counters()
    assert c["jacobians"] == 3 and c["f_points"] == 3 * n
