"""Derivatives with a scalar input per step size on the device, through the C ABI (fdb_derivative / fdb_derivative_complex):
finite_difference_derivative! over arrays (src/derivatives.jl:197-233) and the scalar -> vector finite_difference_gradient!
(src/gradients.jl:477-533).

Every parity assert is a bit compare against the C restatement in scalar_oracle/ (fed the CPU twin of the same synthetic
f), never a tolerance; only the reference's KATs use the reference's tolerances.  Covered: every mode, dir = +-1, step
overrides, sizes around the 1024-element tile, unaligned buffers, batch caps 1 and 2, grids with several tiles per block,
IEEE edges at tile boundaries, every argument f sees, the caller's x left untouched, plan reuse and CUDA-graph replay, and
the rejections."""
import ctypes as C
import math
import re

import numpy as np
import pytest

from _util import assert_same_bits, fdb_env, traced
from scalar_oracle import fd_scalar_oracle as so

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps
FD = {"forward": so.FORWARD, "forward_fx": so.FORWARD, "central": so.CENTRAL, "central_b2": so.CENTRAL,
      "complex": so.COMPLEX}
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1.7e308]
STEP_PAIRS = [(None, None), (0.0, None), (1e-3, 0.0), (-1e-3, 1e-160), (1.0, 5e-324), (0.0, 0.0), (None, 1e-160),
              (1e-3, 5e-324)]


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    so.build()
    so.lib()
    import _bootstrap
    return _bootstrap.load_package()


def _fd_name(mode):
    return {"forward": "forward", "forward_fx": "forward", "central": "central", "central_b2": "central",
            "complex": "complex"}[mode]


class Synth:
    """A native synthetic f (fdbs_poly* / fdbs_tpoly*) with its CPU twin."""

    def __init__(self, pkg, name, n, seed=0, max_batch=1):
        rng = np.random.default_rng(seed)
        self.a, self.w = 0.5 + rng.random(n), rng.random(n) * 2 - 1
        self.d_a = torch.from_numpy(self.a).cuda() if n else torch.zeros(1, dtype=torch.float64, device="cuda")
        self.d_w = torch.from_numpy(self.w).cuda() if n else torch.zeros(1, dtype=torch.float64, device="cuda")
        self.ctx = pkg._lib.ScalarCtx(n, self.d_a.data_ptr(), self.d_w.data_ptr(), 0)
        self.fn = pkg.NativeFn(C.cast(getattr(pkg._lib.synth(), "fdbs_" + name), C.c_void_p).value, self.ctx,
                               max_batch=max_batch, keepalive=(self.d_a, self.d_w))
        self.twin = so.SynthScalar(n, self.a, self.w)
        self.name = name

    def native(self):
        return self.twin.native("synth_" + self.name)


def _x(n, seed, edges=()):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
    for pos, v in edges:
        x[pos] = v
    return x


def _derive(pkg, mode, xh, *, name="poly", relstep=None, absstep=None, dir=1.0, offset=0, cache_kw=None, seed=0):
    """One device derivative of fdbs_<name> at xh and its restatement.  offset = 1 misaligns x, df and fx by one element."""
    n = xh.size
    fd = _fd_name(mode)
    sfx = "_c" if mode == "complex" else ""
    s = Synth(pkg, name + sfx, n, seed)
    xbuf = torch.zeros(n + offset, dtype=torch.float64, device="cuda")
    xbuf[offset:] = torch.from_numpy(xh)
    x = xbuf[offset:]
    fx_t, fx_h = None, None
    if mode == "forward_fx":
        fx_h = np.array([getattr(so.lib(), "synth_" + name)(s.twin.native("synth_" + name)[1], i, xh[i]) for i in range(n)])
        fbuf = torch.zeros(n + offset, dtype=torch.float64, device="cuda")
        fbuf[offset:] = torch.from_numpy(fx_h)
        fx_t = fbuf[offset:]
    kw = dict(cache_kw or {})
    if mode == "central_b2":
        kw["max_batch"] = 2
    cache = pkg.DerivativeCache(x, fx_t, None, fd, **kw)
    dbuf = torch.full((n + offset,), float("nan"), dtype=torch.float64, device="cuda")
    df = dbuf[offset:]
    pkg.finite_difference_derivative_(df, s.fn, x, cache, relstep=relstep, absstep=absstep, dir=dir)
    torch.cuda.synchronize()
    assert_same_bits(x, xh, "caller's x modified")
    ref = so.derivative(s.native(), xh, FD[mode], fx=fx_h, relstep=relstep, absstep=absstep, dir=dir)
    return df, ref, cache, s


def _expected_points(mode):
    return {"forward": 2, "forward_fx": 1, "central": 2, "central_b2": 2, "complex": 1}[mode]


# ------------------------------------------------------------------------------------------------ sizes and modes
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1023, 1024, 1025, 1_000_003])
@pytest.mark.parametrize("mode", list(FD))
def test_gpu_derivative_bitexact(pkg, mode, n):
    xh = _x(n, n)
    df, ref, cache, s = _derive(pkg, mode, xh, seed=n)
    assert_same_bits(df, ref["df"], f"{mode} n={n}")
    c = cache._last_plan.counters()
    assert c["f_points"] == _expected_points(mode) and s.ctx.calls == _expected_points(mode)
    assert c["f_invocations"] == (1 if mode in ("central_b2", "complex", "forward_fx") else 2)
    info = cache._last_plan.info()
    assert info["n_entries"] == n and info["fcalls_per_jacobian"] == _expected_points(mode)
    assert info["alg_bytes_scatter"] == {"forward": 48, "forward_fx": 48, "central": 56, "central_b2": 56,
                                         "complex": 48}[mode] * n


@pytest.mark.parametrize("mode", ["forward", "forward_fx", "central", "central_b2"])
def test_gpu_derivative_step_overrides_and_dir(pkg, mode):
    # one plan reused across every (relstep, absstep, dir): the step scalars are call arguments, not plan state
    n = 1025
    xh = _x(n, 7, [(0, 0.0), (1, -0.0), (1023, 1.0), (1024, -1e-320)])
    s = Synth(pkg, "poly_guarded", n, 3)
    x = torch.from_numpy(xh).cuda()
    fx_h = fx_t = None
    if mode == "forward_fx":
        fx_h = np.array([so.lib().synth_poly_guarded(s.twin.native("synth_poly_guarded")[1], i, xh[i]) for i in range(n)])
        fx_t = torch.from_numpy(fx_h).cuda()
    cache = pkg.DerivativeCache(x, fx_t, None, _fd_name(mode), max_batch=2 if mode == "central_b2" else 1)
    df = torch.empty(n, dtype=torch.float64, device="cuda")
    for relstep in [None, 0.0, 1e-3, -1e-3, 1.0]:
        for absstep in [None, 0.0, 1e-160, 5e-324]:
            for dir in (1.0, -1.0, 0.3):      # |dir| != 1: eps*dir rounds, so x + eps*dir is not one fma
                df.fill_(float("nan"))
                pkg.finite_difference_derivative_(df, s.fn, x, cache, relstep=relstep, absstep=absstep, dir=dir)
                ref = so.derivative(s.native(), xh, FD[mode], fx=fx_h, relstep=relstep, absstep=absstep, dir=dir)
                assert_same_bits(df, ref["df"], f"{mode} relstep={relstep} absstep={absstep} dir={dir}")
    assert_same_bits(x, xh, "caller's x modified")
    assert cache._last_plan.counters()["jacobians"] == 60


@pytest.mark.parametrize("n", [1025, 4099])
@pytest.mark.parametrize("mode", list(FD))
def test_gpu_derivative_unaligned(pkg, mode, n):
    xh = _x(n, 11 + n)
    df, ref, cache, s = _derive(pkg, mode, xh, offset=1, seed=5)
    assert_same_bits(df, ref["df"], f"{mode} unaligned n={n}")


# ------------------------------------------------------------------------------------------------ IEEE edges
@pytest.mark.parametrize("mode", list(FD))
def test_gpu_derivative_ieee_edges_at_tile_boundaries(pkg, mode):
    n = 3000
    positions = [0, 1, 1023, 1024, 1025, 2047, 2048, n - 1]
    for k, v in enumerate(EDGES):
        edges = [(p, EDGES[(k + j) % len(EDGES)]) for j, p in enumerate(positions)]
        xh = _x(n, 100 + k, edges)
        for relstep, absstep in STEP_PAIRS:
            for dir in ((1.0, -1.0) if mode.startswith("forward") else (1.0,)):
                df, ref, cache, s = _derive(pkg, mode, xh, name="poly_guarded", relstep=relstep, absstep=absstep,
                                            dir=dir, seed=k)
                assert_same_bits(df, ref["df"], f"{mode} edges {k} relstep={relstep} absstep={absstep} dir={dir}")
                if mode == "complex":
                    break


def test_gpu_derivative_overflowing_double_step(pkg):
    # relstep = 1 at 1.7e308: x + eps overflows, 2eps overflows and the central reciprocal 1/(2eps) is 0
    xh = np.array([1.7e308, -1.7e308, 1.0, 8.9e307])
    for mode in ("forward", "central"):
        df, ref, _, _ = _derive(pkg, mode, xh, name="poly_guarded", relstep=1.0, absstep=0.0)
        assert_same_bits(df, ref["df"], f"{mode} at 1.7e308")
    assert ref["df"][0] == 0.0


def test_gpu_derivative_zero_steps_on_signed_zeros(pkg):
    # eps = +0.0 (dir = 1) and -0.0 (dir = -1) landing on +-0.0 components: x + (-0.0) keeps -0.0, the guarded f sees it
    xh = np.array([0.0, -0.0] * 20)
    for dir in (1.0, -1.0):
        for mode in ("forward", "forward_fx"):
            df, ref, _, _ = _derive(pkg, mode, xh, name="poly_guarded", relstep=0.0, absstep=0.0, dir=dir)
            assert_same_bits(df, ref["df"], f"{mode} zero step dir={dir}")
    df, ref, _, _ = _derive(pkg, "central", xh, name="poly_guarded", relstep=0.0, absstep=-0.0)
    assert_same_bits(df, ref["df"], "central step -0.0")
    df, ref, _, _ = _derive(pkg, "complex", xh, name="poly_guarded")
    assert_same_bits(df, ref["df"], "complex: the real part of a -0.0 component reads +0.0")


# ------------------------------------------------------------------------------------------------ every argument f sees
class Recorder:
    """Elementwise Python f that records every argument; the values it returns are exact in every mode."""

    def __init__(self, batched=False):
        self.args = []
        self.batched = batched

    def __call__(self, v):
        self.args.append(v.clone())
        return v * 3.0 + v


@pytest.mark.parametrize("mode", list(FD))
def test_gpu_derivative_points_seen(pkg, mode):
    n = 40
    xh = _x(n, 40, [(0, 0.0), (1, -0.0), (2, 1e-320), (3, -5e-324), (39, -0.0)])
    x = torch.from_numpy(xh).cuda()
    fd = _fd_name(mode)
    rec = Recorder(batched=mode == "central_b2")
    fx_h = fx_t = None
    if mode == "forward_fx":
        fx_h = xh * 3.0 + xh
        fx_t = torch.from_numpy(fx_h).cuda()
    cache = pkg.DerivativeCache(x, fx_t, None, fd, max_batch=2 if mode == "central_b2" else 1)
    for relstep, absstep, dir in [(None, None, 1.0), (0.0, 0.0, -1.0), (1e-3, 0.0, -1.0)]:
        rec.args.clear()
        df = pkg.finite_difference_derivative(rec, x, cache, relstep=relstep, absstep=absstep, dir=dir)
        torch.cuda.synchronize()
        f_host = (lambda z: z * 3.0 + z)
        r = so.derivative(f_host, xh, FD[mode], fx=fx_h, relstep=relstep, absstep=absstep, dir=dir, log=True)
        assert_same_bits(df, r["df"], f"{mode} df")
        got = [a.cpu() for a in rec.args]
        if mode == "complex":
            assert len(got) == 1
            ref = np.array(r["points"]).reshape(-1)
            assert_same_bits(torch.view_as_real(got[0]).reshape(-1), ref, "complex points")
            break
        pts = np.array(r["points"])
        if mode == "forward":
            assert len(got) == 2
            assert_same_bits(got[0], pts[0::2], "call 1: x + eps")
            assert_same_bits(got[1], xh, "call 2: x itself")
        elif mode == "forward_fx":
            assert len(got) == 1
            assert_same_bits(got[0], pts, "x + eps")
        elif mode == "central":
            assert len(got) == 2
            assert_same_bits(got[0], pts[0::2], "call 1: x + eps")
            assert_same_bits(got[1], pts[1::2], "call 2: x - eps")
        else:
            assert len(got) == 1 and tuple(got[0].shape) == (2, n)
            assert_same_bits(got[0][0], pts[0::2], "batched row 0: x + eps")
            assert_same_bits(got[0][1], pts[1::2], "batched row 1: x - eps")
    assert_same_bits(x, xh, "caller's x modified")


# ------------------------------------------------------------------------------------------------ plan reuse and graphs
@pytest.mark.parametrize("mode", ["forward", "forward_fx", "central", "central_b2", "complex"])
def test_gpu_derivative_graph_replay(pkg, mode):
    n = 5000
    fd = _fd_name(mode)
    s = Synth(pkg, "poly_guarded" + ("_c" if mode == "complex" else ""), n, 21)
    xh = _x(n, 21, [(0, -0.0), (4999, 0.0)])
    x = torch.from_numpy(xh).cuda()
    fx_h = fx_t = None
    twin_name = "synth_poly_guarded"

    def fxs(xv):
        return np.array([so.lib().synth_poly_guarded(s.twin.native(twin_name)[1], i, xv[i]) for i in range(n)])

    if mode == "forward_fx":
        fx_h = fxs(xh)
        fx_t = torch.from_numpy(fx_h).cuda()
    cache = pkg.DerivativeCache(x, fx_t, None, fd, max_batch=2 if mode == "central_b2" else 1, use_graph=True)
    df = torch.empty(n, dtype=torch.float64, device="cuda")

    def check(what, **kw):
        df.fill_(float("nan"))
        pkg.finite_difference_derivative_(df, s.fn, x, cache, **kw)
        torch.cuda.synchronize()
        ref = so.derivative(s.native(), x.cpu().numpy(), FD[mode], fx=None if fx_t is None else fx_t.cpu().numpy(), **kw)
        assert_same_bits(df, ref["df"], f"{mode}: {what}")

    check("first call")
    check("replay")
    x2 = _x(n, 22, [(1, -0.0), (1024, 0.0)])
    x.copy_(torch.from_numpy(x2))
    if fx_t is not None:
        fx_t.copy_(torch.from_numpy(fxs(x2)))
    check("x (and cache.fx) changed in place")
    if mode == "forward_fx":
        fx_t = torch.from_numpy(fxs(x2) + 1.0).cuda()
        cache.fx = fx_t
        check("a new cache.fx")
    if mode != "complex":
        check("relstep 0", relstep=0.0, absstep=0.0)
        check("relstep -0.0", relstep=-0.0, absstep=-0.0)
        check("dir -1", relstep=0.0, absstep=0.0, dir=-1.0)
        check("new steps", relstep=1e-3, absstep=1e-160, dir=-1.0)
        check("relstep alone", relstep=1e-2, absstep=1e-160, dir=-1.0)
    c = cache._last_plan.counters()
    assert c["f_points"] == c["jacobians"] * _expected_points(mode)


# ------------------------------------------------------------------------------------------------ several tiles per block
@pytest.mark.parametrize("sm", [1, 3])
@pytest.mark.parametrize("mode", ["forward", "central", "complex"])
def test_gpu_derivative_multiwave(pkg, mode, sm):
    n = 1_000_003
    tiles = (n + 1023) // 1024
    xh = _x(n, 77, [(0, -0.0), (1023, np.nan), (1024, np.inf), (n - 1, -0.0)])
    with fdb_env(SM_COUNT=sm):
        holder = {}
        kern = traced(lambda: holder.update(r=_derive(pkg, mode, xh, name="poly_guarded", seed=sm)))
    df, ref, _, _ = holder["r"]
    assert_same_bits(df, ref["df"], f"{mode} SM_COUNT={sm}")
    for name in ("deriv_points", "deriv_quotient"):
        ks = [k for k in kern if re.search(r"\b" + name + r"<", k[0])]
        assert len(ks) == 1, (name, [k[0][:50] for k in kern])
        assert tiles / ks[0][1] >= 3, f"{name}: grid {ks[0][1]} gives {tiles / ks[0][1]:.1f} tiles per block"


# ------------------------------------------------------------------------------------------------ scalar -> vector gradient
def _sgrad(pkg, mode, m, t, *, name="tpoly", relstep=None, absstep=None, dir=1.0, t_tensor=False, offset=0, seed=0,
           cache_kw=None):
    fd = _fd_name(mode)
    s = Synth(pkg, name + ("_c" if mode == "complex" else ""), m, seed)
    fx_h = fx_t = None
    if mode == "forward_fx":
        fx_h = np.zeros(m)
        getattr(so.lib(), "synth_" + name)(s.twin.native("synth_" + name)[1], fx_h.ctypes.data_as(so._f64p), float(t))
        fbuf = torch.zeros(m + offset, dtype=torch.float64, device="cuda")
        fbuf[offset:] = torch.from_numpy(fx_h)
        fx_t = fbuf[offset:]
    dbuf = torch.full((m + offset,), float("nan"), dtype=torch.float64, device="cuda")
    df = dbuf[offset:]
    kw = dict(cache_kw or {})
    if mode == "central_b2":
        kw["max_batch"] = 2
    if fx_t is not None:
        cache = pkg.GradientCache(fx_t, torch.zeros(m, dtype=torch.float64, device="cuda"),
                                  torch.zeros(m, dtype=torch.float64, device="cuda"), float(t), fd, **kw)
    else:
        cache = pkg.GradientCache(df, float(t), fd, **kw)
    x = torch.tensor([t], dtype=torch.float64, device="cuda") if t_tensor else t
    pkg.finite_difference_gradient_(df, s.fn, x, cache, relstep=relstep, absstep=absstep, dir=dir)
    torch.cuda.synchronize()
    if t_tensor:
        assert_same_bits(x, np.array([t]), "caller's t modified")
    ref = so.scalar_gradient(s.native(), t, m, FD[mode], fx=fx_h, relstep=relstep, absstep=absstep, dir=dir)
    return df, ref, cache, s


@pytest.mark.parametrize("m", [0, 1, 33, 1024, 1025, 1_000_003])
@pytest.mark.parametrize("mode", list(FD))
def test_gpu_scalar_gradient_bitexact(pkg, mode, m):
    for t_tensor in (False, True):
        df, ref, cache, s = _sgrad(pkg, mode, m, 0.7318, t_tensor=t_tensor, seed=m)
        assert_same_bits(df, ref["df"], f"{mode} m={m} t_tensor={t_tensor}")
        assert s.ctx.calls == ref["fcalls"] == _expected_points(mode)
        info = cache._last_plan.info()
        assert info["n_entries"] == m and info["fcalls_per_jacobian"] == ref["fcalls"]


@pytest.mark.parametrize("mode", list(FD))
def test_gpu_scalar_gradient_edges_and_steps(pkg, mode):
    m = 1025
    for t in EDGES + [0.25, -3.5]:
        for relstep, absstep in STEP_PAIRS:
            for dir in ((1.0, -1.0, 0.3) if mode.startswith("forward") else (1.0,)):
                for offset in (0, 1):
                    df, ref, _, _ = _sgrad(pkg, mode, m, t, name="tpoly_guarded", relstep=relstep, absstep=absstep,
                                           dir=dir, offset=offset, t_tensor=offset == 1, seed=3)
                    assert_same_bits(df, ref["df"], f"{mode} t={t} relstep={relstep} absstep={absstep} dir={dir}")
            if mode == "complex":
                break


def test_gpu_scalar_gradient_call_order(pkg):
    # f(c1, t + eps) first, then f(c2, t) (forward) or f(c2, t - eps) (central): gradients.jl:495-515
    t = 1.25
    for mode, b2 in (("forward", False), ("central", False), ("central", True)):
        seen = []

        def f(fx, tt):
            seen.append(float(tt))
            fx.copy_(torch.stack([torch.sin(tt), torch.cos(tt)]))

        df = torch.zeros(2, dtype=torch.float64, device="cuda")
        cache = pkg.GradientCache(df, t, mode, max_batch=2 if b2 else 1)
        pkg.finite_difference_gradient_(df, f, t, cache)
        ref = so.scalar_gradient(lambda fx, tt: None, t, 2, FD[mode], log=True)
        assert_same_bits(np.array(seen), np.array(ref["points"]), f"{mode} b2={b2}: arguments in call order")
    seen = []

    def fc(fx, tt):
        seen.append(complex(tt))
        fx.copy_(torch.stack([torch.sin(tt), torch.cos(tt)]))

    pkg.finite_difference_gradient(fc, -0.0, "complex", c1=torch.zeros(2, dtype=torch.float64, device="cuda"))
    assert len(seen) == 1 and math.copysign(1.0, seen[0].real) == 1.0 and seen[0].imag == EPS


@pytest.mark.parametrize("mode", ["forward", "forward_fx", "central", "complex"])
def test_gpu_scalar_gradient_graph_follows_t_in_place(pkg, mode):
    # the ODE use: t lives in device memory and is advanced in place between replays of one captured graph
    m = 4096
    s = Synth(pkg, "tpoly" + ("_c" if mode == "complex" else ""), m, 8)
    t = torch.tensor([0.5], dtype=torch.float64, device="cuda")
    df = torch.empty(m, dtype=torch.float64, device="cuda")
    fx_t = torch.zeros(m, dtype=torch.float64, device="cuda") if mode == "forward_fx" else None
    if fx_t is not None:
        cache = pkg.GradientCache(fx_t, torch.zeros_like(df), torch.zeros_like(df), 0.0, "forward", use_graph=True)
    else:
        cache = pkg.GradientCache(df, 0.0, _fd_name(mode), use_graph=True)
    for k, tv in enumerate([0.5, 0.75, -0.0, 2.0]):
        t.fill_(tv)
        fx_h = None
        if fx_t is not None:
            fx_h = np.zeros(m)
            so.lib().synth_tpoly(s.twin.native("synth_tpoly")[1], fx_h.ctypes.data_as(so._f64p), tv)
            fx_t.copy_(torch.from_numpy(fx_h))
        pkg.finite_difference_gradient_(df, s.fn, t, cache)
        torch.cuda.synchronize()
        ref = so.scalar_gradient(s.native(), tv, m, FD[mode], fx=fx_h)
        assert_same_bits(df, ref["df"], f"{mode} replay {k} at t={tv}")
    c = cache._last_plan.counters()
    assert c["jacobians"] == 4 and c["f_points"] == 4 * _expected_points(mode)
    for relstep, absstep in ((0.0, 0.0), (-0.0, -0.0)):
        if mode == "complex":
            break
        t.fill_(-0.0)
        pkg.finite_difference_gradient_(df, s.fn, t, cache, relstep=relstep, absstep=absstep)
        torch.cuda.synchronize()
        ref = so.scalar_gradient(s.native(), -0.0, m, FD[mode], fx=fx_h, relstep=relstep, absstep=absstep)
        assert_same_bits(df, ref["df"], f"{mode} signed-zero step {relstep}")
    if mode != "complex":
        t.fill_(0.75)
        for relstep in (1e-3, 1e-2):                   # relstep alone changes: a new graph
            pkg.finite_difference_gradient_(df, s.fn, t, cache, relstep=relstep, absstep=1e-160)
            torch.cuda.synchronize()
            ref = so.scalar_gradient(s.native(), 0.75, m, FD[mode], fx=None if fx_t is None else fx_t.cpu().numpy(),
                                     relstep=relstep, absstep=1e-160)
            assert_same_bits(df, ref["df"], f"{mode} relstep {relstep}")


# ------------------------------------------------------------------------------------------------ reference KATs
def err_func(a, b):
    return float((a - b).abs().max())


def test_gpu_kat_derivative(pkg):
    # finitedifftests.jl:10-49 with torch.sin as f
    x = torch.linspace(-2 * math.pi, 2 * math.pi, 100, dtype=torch.float64, device="cuda")
    y = torch.sin(x)
    df_ref = torch.cos(x)
    eps_arr = torch.zeros_like(x)
    for fd, tol in (("forward", 1e-4), ("central", 1e-8), ("complex", 1e-15)):
        assert err_func(pkg.finite_difference_derivative(torch.sin, x, fd), df_ref) < tol
        with pytest.warns(UserWarning) if fd != "forward" else _nullcontext():
            assert err_func(pkg.finite_difference_derivative(torch.sin, x, fd, torch.float64, y, eps_arr), df_ref) < tol
        df = torch.zeros_like(x)
        pkg.finite_difference_derivative_(df, torch.sin, x, fd)
        assert err_func(df, df_ref) < tol
    caches = {"forward": pkg.DerivativeCache(x, y, eps_arr, "forward"),
              "central": pkg.DerivativeCache(x, None, eps_arr, "central"),
              "complex": pkg.DerivativeCache(x, None, None, "complex")}
    for fd, tol in (("forward", 1e-4), ("central", 1e-8), ("complex", 1e-15)):
        df = torch.zeros_like(x)
        pkg.finite_difference_derivative_(df, torch.sin, x, caches[fd])
        assert err_func(df, df_ref) < tol
    assert torch.equal(eps_arr, torch.zeros_like(x))          # the StridedArray path never writes cache.epsilon


class _nullcontext:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def test_gpu_kat_scalar_gradient(pkg):
    # finitedifftests.jl:264-291
    z = x = 2 * math.pi * float(np.random.default_rng(264).random())
    df_ref = torch.tensor([math.cos(x), -math.sin(x)], dtype=torch.float64, device="cuda")

    def f(fx, t):
        fx[0] = torch.sin(t)
        fx[1] = torch.cos(t)

    def ff(fx, t):
        if float(t.real) > z:
            raise RuntimeError("perturbed upward")
        f(fx, t)

    fx = torch.zeros(2, dtype=torch.float64, device="cuda")
    f(fx, torch.tensor(x, dtype=torch.float64, device="cuda"))
    assert err_func(pkg.finite_difference_gradient(f, x, "forward", fx=fx), df_ref) < 1e-4
    assert err_func(pkg.finite_difference_gradient(ff, x, "forward", fx=fx, dir=-1), df_ref) < 1e-4
    with pytest.raises(TypeError):                                   # :277, :280
        pkg.finite_difference_gradient(ff, x, "forward")
    with pytest.raises(RuntimeError, match="perturbed upward"):
        pkg.finite_difference_gradient(ff, x, "forward", fx=fx)
    assert err_func(pkg.finite_difference_gradient(f, x, "central", fx=fx), df_ref) < 1e-8
    assert err_func(pkg.finite_difference_gradient(f, x, "complex", fx=fx), df_ref) < 1e-15
    for fd, tol in (("forward", 1e-4), ("central", 1e-8), ("complex", 1e-15)):
        df = torch.zeros(2, dtype=torch.float64, device="cuda")
        pkg.finite_difference_gradient_(df, f, x, fd)
        assert err_func(df, df_ref) < tol
        df = torch.zeros(2, dtype=torch.float64, device="cuda")
        cache = pkg.GradientCache(df, x, fd)
        pkg.finite_difference_gradient_(df, f, x, cache)
        assert err_func(df, df_ref) < tol


# ------------------------------------------------------------------------------------------------ rejections
def _plan(pkg, create, *args, fdtype=0, world=1):
    L = pkg._lib
    h = C.c_void_p()
    o = L.PlanOpts(fdtype=fdtype, device=0, world=world)
    st = getattr(L.lib(), create)(C.byref(h), *args, C.byref(o))
    return st, h


def test_gpu_derivative_rejections(pkg):
    L = pkg._lib
    lib = L.lib()
    x = torch.rand(8, dtype=torch.float64, device="cuda")
    df = torch.zeros(8, dtype=torch.float64, device="cuda")
    s = Synth(pkg, "poly", 8)
    f = C.c_void_p(s.fn.address)
    nan = float("nan")
    st, dp = _plan(pkg, "fdb_derivative_plan_create", 8)
    assert st == L.FDB_OK
    st, gp = _plan(pkg, "fdb_scalar_gradient_plan_create", 8)
    assert st == L.FDB_OK
    try:
        for p in (dp, gp):
            assert lib.fdb_jacobian(p, f, s.fn.ctx_ptr, x.data_ptr(), df.data_ptr(), None, None, nan, nan, 1.0, None) == L.FDB_ERR_INVALID
            assert lib.fdb_hessian(p, f, s.fn.ctx_ptr, x.data_ptr(), df.data_ptr(), None, nan, nan, None) == L.FDB_ERR_INVALID
            assert lib.fdb_jvp(p, f, s.fn.ctx_ptr, df.data_ptr(), x.data_ptr(), x.data_ptr(), None, None, None, nan, nan, 1.0, None) == L.FDB_ERR_INVALID
            assert lib.fdb_color_eps(p, x.data_ptr(), nan, nan, 1.0, None, None) == L.FDB_ERR_INVALID
            assert lib.fdb_derivative_complex(p, f, s.fn.ctx_ptr, df.data_ptr(), x.data_ptr(), None) == L.FDB_ERR_INVALID
            out = np.zeros(8)
            assert lib.fdb_plan_get_eps(p, out.ctypes.data_as(C.POINTER(C.c_double)), 8, None) == L.FDB_ERR_INVALID
        for create, args in (("fdb_plan_create_dense", (1, 8, 1)), ("fdb_jvp_plan_create", (8, 8))):
            st, other = _plan(pkg, create, *args)
            assert st == L.FDB_OK
            assert lib.fdb_derivative(other, f, s.fn.ctx_ptr, df.data_ptr(), x.data_ptr(), None, nan, nan, 1.0, None) == L.FDB_ERR_INVALID
            lib.fdb_plan_destroy(other)
        st, hp = _plan(pkg, "fdb_hessian_plan_create", 8, 8, fdtype=L.FDB_HCENTRAL)
        assert st == L.FDB_OK
        assert lib.fdb_derivative(hp, f, s.fn.ctx_ptr, df.data_ptr(), x.data_ptr(), None, nan, nan, 1.0, None) == L.FDB_ERR_INVALID
        lib.fdb_plan_destroy(hp)
        st, cp = _plan(pkg, "fdb_derivative_plan_create", 8, fdtype=L.FDB_COMPLEX)
        assert st == L.FDB_OK
        assert lib.fdb_derivative(cp, f, s.fn.ctx_ptr, df.data_ptr(), x.data_ptr(), None, nan, nan, 1.0, None) == L.FDB_ERR_INVALID
        lib.fdb_plan_destroy(cp)
    finally:
        lib.fdb_plan_destroy(dp)
        lib.fdb_plan_destroy(gp)
    for create in ("fdb_derivative_plan_create", "fdb_scalar_gradient_plan_create"):
        assert _plan(pkg, create, 8, fdtype=L.FDB_HCENTRAL)[0] == L.FDB_ERR_UNSUPPORTED
        assert _plan(pkg, create, 8, world=2)[0] == L.FDB_ERR_UNSUPPORTED
    # the Python mirror: complex arrays, non-contiguous arrays and CPU tensors are rejected loudly
    with pytest.raises(TypeError):
        pkg.finite_difference_derivative(torch.sin, x.to(torch.complex128))
    with pytest.raises(TypeError):
        pkg.finite_difference_derivative(torch.sin, x.cpu())
    with pytest.raises(ValueError):
        pkg.finite_difference_derivative(torch.sin, torch.rand(8, 2, dtype=torch.float64, device="cuda").t())
    with pytest.raises(TypeError):
        pkg.finite_difference_derivative_(torch.zeros(8, dtype=torch.complex128, device="cuda"), torch.sin, x)
    with pytest.raises(ValueError):
        pkg.DerivativeCache(x, None, None, "complex", torch.complex128)
    with pytest.raises(TypeError):
        pkg.finite_difference_gradient_(torch.zeros(2, dtype=torch.complex128, device="cuda"), lambda fx, t: None, 1.0)
    with pytest.raises(TypeError):
        pkg.finite_difference_gradient_(torch.zeros(2, dtype=torch.float64), lambda fx, t: None, 1.0)
    with pytest.raises(TypeError):
        pkg.finite_difference_gradient_(df, lambda fx, t: None, 1.0 + 2.0j)
    with pytest.raises(ValueError):
        pkg.finite_difference_gradient_(torch.zeros(4, 2, dtype=torch.float64, device="cuda").t(), lambda fx, t: None, 1.0)
