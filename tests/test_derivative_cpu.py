"""Scalar-input derivatives on the CPU: the C restatements of finite_difference_derivative! (src/derivatives.jl:197-233)
and of the scalar -> vector finite_difference_gradient! (src/gradients.jl:477-533) in scalar_oracle/.

- bit for bit against an independent Python transcription written here: df, every argument f sees, call count and order,
  over random x with IEEE edge values, every mode, dir = +-1 and overridden step sizes;
- the CPU twins of the synthetic functions against a numpy evaluation;
- the reference's own KATs (test/finitedifftests.jl:10-49, :264-291) at their tolerances."""
import cmath
import math

import numpy as np
import pytest

from _util import assert_same_bits
from scalar_oracle import fd_scalar_oracle as so

f64 = np.float64
EPS = np.finfo(float).eps
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1.7e308, 1.0]
RELSTEPS = [None, 0.0, 1e-3, -1e-3, 1.0]
ABSSTEPS = [None, 0.0, 1e-160, 5e-324]


@pytest.fixture(scope="module")
def soracle():
    so.build()
    so.lib()
    return so


# ------------------------------------------------------------------------------------------------ transcription
def _max(a, b):                                     # Julia Base.max on Float64
    if math.isnan(a) or math.isnan(b):
        return f64(a - b)
    return b if math.copysign(1.0, a - b) < 0 else a


def _defaults(fd, relstep, absstep):
    rel = {0: f64(np.sqrt(EPS)), 1: f64(np.cbrt(EPS))}[fd] if relstep is None else f64(relstep)
    return rel, (rel if absstep is None else f64(absstep))


def _eps(fd, x, rel, ab, dir):                      # compute_epsilon, epsilons.jl:26-29 / :50-53
    e = _max(rel * f64(abs(x)), ab)
    return f64(e * f64(dir)) if fd == 0 else f64(e)


def derivative_transcribed(f, x, fd, fx, relstep, absstep, dir):
    """derivatives.jl:206-228, line by line; f(i, v) -> float.  Returns (df, arguments in call order)."""
    pts, df = [], np.zeros(len(x))
    with np.errstate(all="ignore"):
        if fd == 2:
            for i in range(len(x)):
                z = (f64(x[i]) + f64(0.0), f64(EPS))              # x[i] + im*eps: im*eps = Complex(0.0, eps)
                pts.append(z)
                df[i] = f64(f(i, z)[1]) / f64(EPS)
            return df, pts
        rel, ab = _defaults(fd, relstep, absstep)
        for i in range(len(x)):
            xi = f64(x[i])
            e = _eps(fd, xi, rel, ab, dir)
            if fd == 0:
                xp = xi + e
                pts.append(xp)
                fp = f64(f(i, xp))
                if fx is None:
                    pts.append(xi)
                    fb = f64(f(i, xi))
                else:
                    fb = f64(fx[i])
                df[i] = (fp - fb) / e
            else:
                inv = f64(1.0) / (f64(2.0) * e)
                xp, xm = xi + e, xi - e
                pts.append(xp)
                fp = f64(f(i, xp))
                pts.append(xm)
                fm = f64(f(i, xm))
                df[i] = (fp - fm) * inv
    return df, pts


def scalar_gradient_transcribed(f, x, m, fd, fx, relstep, absstep, dir):
    """gradients.jl:494-528, line by line; f(t) -> m values (complex: t a (re, im) pair, values complex)."""
    pts = []
    x = f64(x)
    with np.errstate(all="ignore"):
        if fd == 2:
            z = (x + f64(0.0), f64(EPS))
            pts.append(z)
            c1 = f(z)
            return np.array([f64(np.imag(c)) / f64(EPS) for c in c1]), pts
        rel, ab = _defaults(fd, relstep, absstep)
        e = _eps(fd, x, rel, ab, dir)
        pts.append(x + e)
        c1 = np.asarray(f(x + e), dtype=np.float64)
        if fd == 0:
            if fx is not None:
                return (c1 - np.asarray(fx)) / e, pts
            pts.append(x)
            c2 = np.asarray(f(x), dtype=np.float64)
            return (c1 - c2) / e, pts
        pts.append(x - e)
        c2 = np.asarray(f(x - e), dtype=np.float64)
        return (c1 - c2) / (f64(2.0) * e), pts


# ------------------------------------------------------------------------------------------------ synthetic twins
def _poly_np(a, w, v, guarded):
    with np.errstate(all="ignore"):
        q = v * v
        c = q * v
        if not guarded:
            return (a * c + w * q) + v
        g = lambda t, k: np.where(np.isfinite(t) & (np.abs(t) <= 2.0 ** 500), t, k)
        t = (g(a * c, 0.25) + g(w * q, -0.5)) + g(v, 0.75)
        return t + np.where(~np.isnan(v) & np.signbit(v), w, 0.0)


def _problem(n, seed):
    rng = np.random.default_rng(seed)
    return so.SynthScalar(n, 0.5 + rng.random(n), rng.random(n) * 2 - 1)


def test_synth_poly_twins_match_numpy(soracle):
    n = 257
    tw = _problem(n, 1)
    L = soracle.lib()
    rng = np.random.default_rng(2)
    v = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
    v[:len(EDGES)] = EDGES
    for name, g in (("synth_poly", False), ("synth_poly_guarded", True)):
        got = np.array([getattr(L, name)(tw.native(name)[1], i, v[i]) for i in range(n)])
        assert_same_bits(got, _poly_np(tw.a, tw.w, v, g), name)
    out = np.zeros(n)
    L.synth_tpoly_guarded(tw.native("synth_tpoly_guarded")[1], out.ctypes.data_as(so._f64p), -0.0)
    assert_same_bits(out, _poly_np(tw.a, tw.w, np.full(n, -0.0), True), "synth_tpoly_guarded at -0.0")


# ------------------------------------------------------------------------------------------------ restatement vs transcription
def _native_elem(tw, name):
    L = so.lib()
    fn = getattr(L, name)
    ctx = tw.native(name)[1]
    if name.endswith("_c"):
        def f(i, z):
            out = np.zeros(2)
            zz = np.array(z, dtype=np.float64)
            fn(ctx, i, zz.ctypes.data_as(so._f64p), out.ctypes.data_as(so._f64p))
            return out
        return f
    return lambda i, v: fn(ctx, i, float(v))


def _native_vec(tw, name, m):
    L = so.lib()
    fn = getattr(L, name)
    ctx = tw.native(name)[1]
    if name.endswith("_c"):
        def f(z):
            out = np.zeros(2 * m)
            zz = np.array(z, dtype=np.float64)
            fn(ctx, out.ctypes.data_as(so._f64p), zz.ctypes.data_as(so._f64p))
            return out.view(np.complex128)
        return f

    def f(t):
        out = np.zeros(m)
        fn(ctx, out.ctypes.data_as(so._f64p), float(t))
        return out
    return f


def _same_points(got, ref, what):
    assert len(got) == len(ref), f"{what}: {len(got)} f calls, expected {len(ref)}"
    assert_same_bits(np.array(got, dtype=np.float64).reshape(-1), np.array(ref, dtype=np.float64).reshape(-1),
                     f"{what}: f arguments")


@pytest.mark.parametrize("fd", [0, 1, 2])
def test_derivative_restatement_matches_transcription(soracle, fd):
    rng = np.random.default_rng(197 + fd)
    for trial in range(60):
        n = int(rng.integers(0, 40))
        tw = _problem(n, trial)
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
        for k in range(n):
            if rng.random() < 0.3:
                x[k] = EDGES[rng.integers(len(EDGES))]
        relstep = RELSTEPS[rng.integers(len(RELSTEPS))]
        absstep = ABSSTEPS[rng.integers(len(ABSSTEPS))]
        dir = [1.0, -1.0, 0.3][rng.integers(3)]
        name = "synth_poly_guarded" + ("_c" if fd == 2 else "")
        fx = None
        if fd == 0 and rng.random() < 0.5:
            fx = np.array([soracle.lib().synth_poly_guarded(tw.native(name)[1], i, x[i]) for i in range(n)])
        df, pts = derivative_transcribed(_native_elem(tw, name), x, fd, fx, relstep, absstep, dir)
        r = soracle.derivative(tw.native(name), x, fd, fx=fx, relstep=relstep, absstep=absstep, dir=dir, log=True)
        what = f"trial {trial} fd={fd} rel={relstep} abs={absstep} dir={dir} fx={fx is not None}"
        assert r["fcalls"] == len(pts), what
        _same_points(r["points"], pts, what)
        assert_same_bits(r["df"], df, what)


@pytest.mark.parametrize("fd", [0, 1, 2])
def test_scalar_gradient_restatement_matches_transcription(soracle, fd):
    rng = np.random.default_rng(477 + fd)
    for trial in range(80):
        m = int(rng.integers(0, 20))
        tw = _problem(m, 1000 + trial)
        t = EDGES[rng.integers(len(EDGES))] if rng.random() < 0.4 else float(rng.standard_normal() * 10.0 ** rng.integers(-3, 4))
        relstep = RELSTEPS[rng.integers(len(RELSTEPS))]
        absstep = ABSSTEPS[rng.integers(len(ABSSTEPS))]
        dir = [1.0, -1.0, 0.3][rng.integers(3)]
        name = "synth_tpoly_guarded" + ("_c" if fd == 2 else "")
        f = _native_vec(tw, name, m)
        fx = f(t) if fd == 0 and rng.random() < 0.5 else None
        df, pts = scalar_gradient_transcribed(f, t, m, fd, fx, relstep, absstep, dir)
        r = soracle.scalar_gradient(tw.native(name), t, m, fd, fx=fx, relstep=relstep, absstep=absstep, dir=dir, log=True)
        what = f"trial {trial} fd={fd} t={t} rel={relstep} abs={absstep} dir={dir} fx={fx is not None}"
        assert r["fcalls"] == len(pts), what
        _same_points(r["points"], pts, what)
        assert_same_bits(r["df"], df, what)


def test_signed_zero_steps(soracle):
    # eps = 0 with dir = -1 is -0.0: x + (-0.0) keeps a -0.0 component negative; the complex point reads +0.0
    r = soracle.derivative(lambda v: v, np.array([-0.0, 0.0]), so.FORWARD, relstep=0.0, absstep=0.0, dir=-1.0, log=True)
    assert [math.copysign(1.0, p) for p in r["points"]] == [-1.0, -1.0, 1.0, 1.0]
    r = soracle.derivative(lambda v: v, np.array([-0.0]), so.FORWARD, relstep=0.0, absstep=0.0, dir=1.0, log=True)
    assert math.copysign(1.0, r["points"][0]) == 1.0            # -0.0 + (+0.0) = +0.0
    r = soracle.derivative(lambda z: z, np.array([-0.0]), so.COMPLEX, log=True)
    assert math.copysign(1.0, r["points"][0][0]) == 1.0 and r["points"][0][1] == EPS


def test_central_reciprocal_differs_from_division(soracle):
    # the derivative's (f+ - f-) * (1/(2eps)) and the gradient's (c1 - c2) / (2eps) round differently for most eps
    x = np.random.default_rng(9).standard_normal(200)
    d = soracle.derivative(np.sin, x, so.CENTRAL)["df"]
    g = np.array([soracle.scalar_gradient(lambda fx, t: fx.__setitem__(0, np.sin(t)), v, 1, so.CENTRAL)["df"][0] for v in x])
    assert np.count_nonzero(d != g) > 20


# ------------------------------------------------------------------------------------------------ reference KATs
def err_func(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))))


def test_kat_derivative_strided(soracle):
    # finitedifftests.jl:10-49
    x = np.linspace(-2 * np.pi, 2 * np.pi, 100)
    y = np.sin(x)
    df_ref = np.cos(x)
    assert err_func(soracle.derivative(np.sin, x, so.FORWARD)["df"], df_ref) < 1e-4
    assert err_func(soracle.derivative(np.sin, x, so.CENTRAL)["df"], df_ref) < 1e-8
    assert err_func(soracle.derivative(cmath.sin, x, so.COMPLEX)["df"], df_ref) < 1e-15
    r = soracle.derivative(np.sin, x, so.FORWARD, fx=y)                 # forward_cache = DerivativeCache(x, y, epsilon, ..)
    assert err_func(r["df"], df_ref) < 1e-4 and r["fcalls"] == 100
    assert soracle.derivative(np.sin, x, so.FORWARD)["fcalls"] == 200
    assert soracle.derivative(np.sin, x, so.CENTRAL)["fcalls"] == 200
    assert soracle.derivative(cmath.sin, x, so.COMPLEX)["fcalls"] == 100


def test_kat_scalar_gradient(soracle):
    # finitedifftests.jl:264-291: f(df, x) = [sin x, cos x]
    z = x = 2 * np.pi * np.random.default_rng(264).random()
    df_ref = np.array([np.cos(x), -np.sin(x)])

    def f(fx, t):
        fx[0], fx[1] = np.sin(t), np.cos(t)

    def fc(fx, t):
        fx[0], fx[1] = cmath.sin(t), cmath.cos(t)

    r = soracle.scalar_gradient(f, x, 2, so.FORWARD)
    assert err_func(r["df"], df_ref) < 1e-4 and r["fcalls"] == 2       # :278: fx only sizes df, f(x) still runs
    r = soracle.scalar_gradient(f, x, 2, so.FORWARD, dir=-1.0, log=True)   # :279, ff errors for t > z
    assert err_func(r["df"], df_ref) < 1e-4 and all(p <= z for p in r["points"])
    assert err_func(soracle.scalar_gradient(f, x, 2, so.CENTRAL)["df"], df_ref) < 1e-8
    assert err_func(soracle.scalar_gradient(fc, x, 2, so.COMPLEX)["df"], df_ref) < 1e-15
    fx = np.array([np.sin(x), np.cos(x)])
    r = soracle.scalar_gradient(f, x, 2, so.FORWARD, fx=fx)
    assert err_func(r["df"], df_ref) < 1e-4 and r["fcalls"] == 1


def test_scalar_gradient_without_size_is_an_error():
    # finitedifftests.jl:277 (@test_broken) / :280: the cache-less scalar -> vector call with none of fx, c1, c2 cannot
    # size df (gradients.jl:185-186); the check runs before any device work
    import _bootstrap
    pkg = _bootstrap.load_package()
    with pytest.raises(TypeError, match="at least one of fx, c1 or c2"):
        pkg.finite_difference_gradient(lambda fx, t: None, 1.0, "forward")
