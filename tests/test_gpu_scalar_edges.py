"""IEEE edge inputs, overridden step sizes, tile-boundary sizes and graph replay for the device Hessian and gradient.

x holds signed zeros, NaN, +-Inf, subnormals and magnitudes near the ends of the fp64 range; relstep and absstep run
through 0, negative, tiny and subnormal values, chosen so that eps = 0 lands on a +-0.0 component, eps_i * eps_j
underflows where (4 eps_i) * eps_j does not, and eps_i * eps_i overflows.  The function is fdbs_guarded (finite for every
input and sensitive to the sign of a zero) or, where every point f sees is compared, the same function evaluated on the
host.  Every result is bit-compared (tests/_util.assert_same_bits: signed zeros differ, NaN is one class) with the C
restatement's own run (scalar_oracle/), with no tolerance; f-call counts are exact."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, fdb_env, guarded_numpy, max_julia
from scalar_oracle import fd_scalar_oracle as so

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

f64 = np.float64
NAN = float("nan")
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1e-160, 1.0, -2.5]
# (relstep, absstep, first EDGES index placed in x); None = keyword not given
STEPS = [
    (None, None, 8),        # 1e300 with the default step: eps_i * eps_i overflows
    (None, 0.0, 0),         # eps = 0 on the +-0.0 components
    (0.0, None, 1),         # eps = 0 everywhere (absstep defaults to relstep)
    (1e-3, 1e-6, 3),
    (1e-12, 1e-160, 10),
    (None, 1e-320, 5),      # eps_i * eps_j flushed to 0 where (4 eps_i) * eps_j is not
    (-1e-3, None, 0),       # negative relstep: max(-1e-3 |x_i|, -1e-3) decides
    (1e-3, 5e-324, 6),
]
TILE_EDGES = (0, 31, 32, 33)      # plus n - 1: both sides of the first 32-wide assembly tile boundary


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    so.build()
    so.lib()
    import _bootstrap
    return _bootstrap.load_package()


class Guarded:
    """fdbs_guarded on the device, its CPU twin synth_guarded, and the same f evaluated on the host (guarded_numpy)."""

    def __init__(self, pkg, n):
        rng = np.random.default_rng(4000 + n)
        self.n = n
        self.a = 0.5 + rng.random(n)
        self.w = rng.random(n) * 2 - 1
        self.d_a = torch.from_numpy(self.a).cuda()
        self.d_w = torch.from_numpy(self.w).cuda()
        self.ctx = pkg._lib.ScalarCtx(n, self.d_a.data_ptr(), self.d_w.data_ptr(), 0)
        self.fn = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_guarded, C.c_void_p).value, self.ctx,
                               keepalive=(self.d_a, self.d_w))
        self.twin = so.SynthScalar(n, self.a, self.w, name="synth_guarded")

    def host(self, v):
        return float(guarded_numpy(v, self.a, self.w))


def edge_x(n, first, where):
    """ordinary values of both signs; the components in `where` take EDGES[first], EDGES[first + 1], ... in turn"""
    rng = np.random.default_rng(77 + 13 * first + n)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-2, 3, n)
    for r, k in enumerate(sorted({k for k in where if 0 <= k < n})):
        x[k] = EDGES[(first + r) % len(EDGES)]
    return x


def _step_sizes(x, relstep, absstep):
    relstep = f64(2.0 ** -13) if relstep is None else f64(relstep)
    absstep = relstep if absstep is None else f64(absstep)
    with np.errstate(all="ignore"):
        return np.array([max_julia(relstep * abs(v), absstep) for v in x])


def _denominator_order_matters(x, relstep, absstep):
    e = _step_sizes(x, relstep, absstep)
    with np.errstate(all="ignore"):
        p, q = (f64(4) * e[:, None]) * e[None, :], f64(4) * (e[:, None] * e[None, :])
    return bool(np.any((p.view(np.uint64) != q.view(np.uint64)) & ~(np.isnan(p) & np.isnan(q))))


def _cuda(xh):
    return torch.from_numpy(np.array(xh, dtype=np.float64)).cuda()


# ------------------------------------------------------------------------------------------------ Hessian: points f sees
@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("max_batch", [1, 3, 64])
@pytest.mark.parametrize("n", [1, 2, 5, 8])
def test_gpu_hessian_points_seen_by_f_edges(pkg, n, max_batch, batched):
    # a host-evaluated Python f returning a Python float: every point hess_patch builds (steps and restores, signed zeros
    # included) is compared with the restatement's, in call order
    g = Guarded(pkg, n)
    seen = []
    if batched:
        def f(X):
            Xh = X.cpu().numpy().copy()
            seen.extend(Xh)
            return [g.host(r) for r in Xh]
        f.batched = True
    else:
        def f(v):
            vh = v.cpu().numpy().copy()
            seen.append(vh)
            return g.host(vh)
    for relstep, absstep, first in STEPS:
        xh = edge_x(n, first, range(0, n, 2))
        x = _cuda(xh)
        what = f"n={n} max_batch={max_batch} batched={batched} relstep={relstep} absstep={absstep} x={xh}"
        ref = so.hessian(g.host, xh, relstep=relstep, absstep=absstep, log=True)
        seen.clear()
        H = pkg.zeros_colmajor(n, n)
        fx = torch.full((1,), NAN, dtype=torch.float64, device="cuda")
        cache = pkg.HessianCache(x, max_batch=max_batch)
        pkg.finite_difference_hessian_(H, f, x, cache, relstep=relstep, absstep=absstep, fx=fx)
        torch.cuda.synchronize()
        assert len(seen) == len(ref["points"]) == 2 * n * n + 1, what
        for k, (p, q) in enumerate(zip(seen, ref["points"])):
            assert_same_bits(p, q, f"{what}: point {k}")
        assert_same_bits(H, ref["H"][:n, :n], f"{what}: H")
        assert_same_bits(fx, np.array([ref["fx"]]), f"{what}: f(x)", allow_nan=False)
        assert_same_bits(x, xh, f"{what}: x modified")
        assert cache._last_plan.counters()["f_points"] == 2 * n * n + 1


# ------------------------------------------------------------------------------------------------ Hessian: native f, tile edges
def _block_start(i, n):
    return 1 + 2 * i + 4 * (i * (n - 1) - i * (i - 1) // 2)


def _chunk_bounds(n, max_batch, scratch_bytes):
    """fdb_hessian_plan_create's rule, restated: the batch rows take at most half the budget, and each chunk is the
    longest run of whole i-blocks (at least one) whose values fit what is left, less one slot for f(x)."""
    ldx = max(2, (n + 1) & ~1)
    total = 2 * n * n + 1
    budget = scratch_bytes if scratch_bytes > 0 else 8 << 30
    batch = max(1, min(max(max_batch, 1), budget // 2 // (8 * ldx)))
    batch = min(batch, total, 4096)
    cap = max((budget - batch * ldx * 8) // 8 - 1, 0)
    bounds, i0 = [0], 0
    while i0 < n:
        i1 = i0 + 1
        while i1 < n and _block_start(i1 + 1, n) - _block_start(i0, n) <= cap:
            i1 += 1
        bounds.append(i1)
        i0 = i1
    return bounds


def _scratch_first_chunk(n, max_batch, i_end):
    """the budget whose first chunk is exactly the i-blocks [0, i_end)"""
    ldx = max(2, (n + 1) & ~1)
    scratch = max_batch * ldx * 8 + 8 * (1 + _block_start(i_end, n) - _block_start(0, n))
    assert scratch // 2 // (8 * ldx) >= max_batch            # the batch keeps its cap under this budget
    bounds = _chunk_bounds(n, max_batch, scratch)
    assert bounds[1] == i_end and len(bounds) > 2, bounds
    return scratch


_ORACLE = {}


def _oracle_hessian(g, xh, relstep, absstep):
    key = (g.n, xh.tobytes(), repr(relstep), repr(absstep))
    if key not in _ORACLE:
        _ORACLE[key] = so.hessian(g.twin.native("synth_guarded"), xh, relstep=relstep, absstep=absstep)
    return _ORACLE[key]


def _device_hessian(pkg, g, x, cache, relstep, absstep, ld):
    n = g.n
    buf = torch.full((n, ld), NAN, dtype=torch.float64, device="cuda")     # column j of H = buf[j]
    H = buf[:, :n].t()
    fx = torch.full((1,), NAN, dtype=torch.float64, device="cuda")
    pkg.finite_difference_hessian_(H, g.fn, x, cache, relstep=relstep, absstep=absstep, fx=fx)
    torch.cuda.synchronize()
    return H, buf, fx


HCASES = ["max_batch 7", "max_batch 4096", "chunk at i=32", "chunk mid-tile", "ldH n+1", "ldH n+31", "FDB_SM_COUNT=1"]


@pytest.mark.parametrize("n,case", [(n, c) for n in (31, 32, 33, 64, 65, 97) for c in HCASES
                                    if not (c == "chunk at i=32" and n <= 32)])
def test_gpu_hessian_native_edges(pkg, n, case):
    g = Guarded(pkg, n)
    max_batch = 4096 if case == "max_batch 4096" else 7
    ld = {"ldH n+1": n + 1, "ldH n+31": n + 31}.get(case, n)
    scratch = {"chunk at i=32": lambda: _scratch_first_chunk(n, 7, 32),
               "chunk mid-tile": lambda: _scratch_first_chunk(n, 7, 16)}.get(case, lambda: 0)()
    kw = {"scratch_bytes": scratch} if scratch else {}
    with fdb_env(SM_COUNT=1 if case == "FDB_SM_COUNT=1" else None):
        cache = pkg.HessianCache(torch.zeros(n, dtype=torch.float64, device="cuda"), max_batch=max_batch, **kw)
        for k, (relstep, absstep, first) in enumerate(STEPS):
            xh = edge_x(n, first, TILE_EDGES + (n - 1,))
            if (relstep, absstep) == (None, 1e-320):
                assert _denominator_order_matters(xh, relstep, absstep)
            x = _cuda(xh)
            what = f"n={n} {case} relstep={relstep} absstep={absstep}"
            ref = _oracle_hessian(g, xh, relstep, absstep)
            g.ctx.calls = 0
            H, buf, fx = _device_hessian(pkg, g, x, cache, relstep, absstep, ld)
            assert_same_bits(H, ref["H"][:n, :n], f"{what}: H")
            assert_same_bits(fx, np.array([ref["fx"]]), f"{what}: f(x)", allow_nan=False)
            assert_same_bits(x, xh, f"{what}: x modified")
            plan = cache._last_plan
            assert g.ctx.calls == ref["fcalls"] == 2 * n * n + 1
            assert plan.counters()["f_points"] == (k + 1) * (2 * n * n + 1)
            if ld > n:
                assert torch.isnan(buf[:, n:]).all(), f"{what}: padding rows beyond n were written"
    info = plan.info()
    if scratch:
        assert info["n_groups"] == len(_chunk_bounds(n, max_batch, scratch)) - 1
    else:
        assert info["n_groups"] == 1


def test_gpu_hessian_edges_reach_overflow_and_zero_steps():
    # the step-size edges STEPS promises, checked on the inputs the native test builds
    for n in (33, 97):
        x = edge_x(n, 8, TILE_EDGES + (n - 1,))
        e = _step_sizes(x, None, None)
        with np.errstate(over="ignore"):
            assert np.isinf(e[0] * e[0]) and np.isfinite(e[0])                  # x[0] = 1e300
        x = edge_x(n, 0, TILE_EDGES + (n - 1,))
        e = _step_sizes(x, None, 0.0)
        assert e[0] == 0 and e[31] == 0 and np.signbit(x[31])                    # x[0] = +0.0, x[31] = -0.0


# ------------------------------------------------------------------------------------------------ Hessian: graph replay
def test_gpu_hessian_graph_replay_follows_x_and_steps(pkg):
    # use_graph: a call with the same arguments replays the captured graph, which reads x where it lies (x changed in
    # place is followed); a call with other step sizes is a different call and recaptures.  The native f's host side
    # runs only while a graph is captured, so ctx.calls tells a recapture (2n^2 + 1 more) from a replay (none).
    n = 33
    g = Guarded(pkg, n)
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    buf = torch.full((n, n), NAN, dtype=torch.float64, device="cuda")
    H = buf.t()
    fx = torch.full((1,), NAN, dtype=torch.float64, device="cuda")
    cache = pkg.HessianCache(x, max_batch=64, use_graph=True)
    seq = [(8, None, None, True), (5, None, None, False), (5, 1e-3, None, True), (5, 1e-3, 1e-6, True),
           (1, 1e-3, 1e-6, False), (1, 0.0, 0.0, True), (1, -0.0, -0.0, True), (1, 0.0, 0.0, True)]
    total = 2 * n * n + 1
    for k, (first, relstep, absstep, captured) in enumerate(seq):
        xh = edge_x(n, first, TILE_EDGES + (n - 1,))
        x.copy_(_cuda(xh))                                     # same storage, new values
        calls0 = g.ctx.calls
        pkg.finite_difference_hessian_(H, g.fn, x, cache, relstep=relstep, absstep=absstep, fx=fx)
        torch.cuda.synchronize()
        what = f"call {k}: x from EDGES[{first}], relstep={relstep} absstep={absstep}"
        ref = so.hessian(g.twin.native("synth_guarded"), xh, relstep=relstep, absstep=absstep)
        assert_same_bits(H, ref["H"], f"{what}: H")
        assert_same_bits(fx, np.array([ref["fx"]]), f"{what}: f(x)", allow_nan=False)
        assert g.ctx.calls - calls0 == (total if captured else 0), f"{what}: {'not ' if captured else ''}recaptured"
        c = cache._last_plan.counters()
        assert c["jacobians"] == k + 1 and c["f_points"] == (k + 1) * total


# ------------------------------------------------------------------------------------------------ gradient: native f
GMODES = ["forward", "forward, fx number", "forward, fx tensor", "central", "forward, dir=-1"]


def _expected_calls(mode, n):
    return 2 * n if mode == "central" else (n if "fx" in mode else n + 1)


@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("max_batch", [1, 64])
@pytest.mark.parametrize("mode", GMODES)
@pytest.mark.parametrize("n", [1, 7, 33, 1000])
def test_gpu_gradient_native_edges(pkg, n, mode, max_batch, aligned):
    g = Guarded(pkg, n)
    fd = "central" if mode == "central" else "forward"
    code = so.CENTRAL if mode == "central" else so.FORWARD
    dir = -1.0 if mode == "forward, dir=-1" else 1.0
    store = torch.empty(n + 1, dtype=torch.float64, device="cuda")
    x = store[:n] if aligned else store[1:]                   # unaligned: a view at element offset 1
    fx_t = torch.full((1,), NAN, dtype=torch.float64, device="cuda")
    if "fx" in mode:
        cache = pkg.GradientCache(fx_t if "tensor" in mode else 0.0, None, None, torch.zeros(n, dtype=torch.float64,
                                  device="cuda"), fd, max_batch=max_batch)
    else:
        cache = pkg.GradientCache(torch.zeros(n, dtype=torch.float64, device="cuda"), x, fd, max_batch=max_batch)
    df = torch.full((n,), NAN, dtype=torch.float64, device="cuda")
    for relstep, absstep, first in STEPS:
        xh = edge_x(n, first, TILE_EDGES + (n - 1,))
        x.copy_(_cuda(xh))
        fxv = None
        if "fx" in mode:
            fxv = g.twin(xh)
            if "tensor" in mode:
                fx_t.fill_(fxv)
            else:
                cache.fx = fxv                                 # a new number for every call
        what = f"n={n} {mode} max_batch={max_batch} aligned={aligned} relstep={relstep} absstep={absstep}"
        g.ctx.calls = 0
        pkg.finite_difference_gradient_(df, g.fn, x, cache, relstep=relstep, absstep=absstep, dir=dir)
        torch.cuda.synchronize()
        ref = so.gradient(g.twin.native("synth_guarded"), xh, code, fx=fxv, relstep=relstep, absstep=absstep, dir=dir)
        assert_same_bits(df, ref["df"], f"{what}: df")
        assert g.ctx.calls == ref["fcalls"] == _expected_calls(mode, n), what
        assert_same_bits(x, xh, f"{what}: x modified")


# ------------------------------------------------------------------------------------------------ gradient: complex step
def guarded_complex(z, a, w):
    """fdbs_guarded's formula on complex128 values, written out on numpy scalars (host only: the same function runs
    for the device's calls and the restatement's); g replaces a term whose parts are not finite or exceed 2^500"""
    def g(t, c):
        ok = np.isfinite(t.real) and np.isfinite(t.imag) and abs(t.real) <= 2.0 ** 500 and abs(t.imag) <= 2.0 ** 500
        return t if ok else np.complex128(c)

    n = len(z)
    s1 = s2 = np.complex128(0)
    with np.errstate(all="ignore"):
        for k in range(n):
            v = z[k]
            t = g(a[k] * (v * v * v * v), 0.25)
            if k + 1 < n:
                t = t + g(v * z[k + 1], -0.5)
            if not np.isnan(v.real) and np.signbit(v.real):
                t = t + w[k]
            s1 = s1 + t
            s2 = s2 + g(w[k] * v, 0.75)
        s = g(s2, 1.5)
        return complex(s1 + (s * s) / np.float64(2 * n))


@pytest.mark.parametrize("max_batch", [1, 64])
@pytest.mark.parametrize("n", [1, 2, 5, 8])
def test_gpu_gradient_complex_points_edges(pkg, n, max_batch):
    g = Guarded(pkg, n)
    seen = []

    def f(z):
        zh = z.cpu().numpy().copy()
        seen.append(zh.view(np.float64).copy())
        return guarded_complex(zh, g.a, g.w)

    for first in range(len(EDGES)):
        xh = edge_x(n, first, range(0, n, 2))
        x = _cuda(xh)
        what = f"n={n} max_batch={max_batch} x={xh}"
        ref = so.gradient(lambda z: guarded_complex(z, g.a, g.w), xh, so.COMPLEX, log=True)
        seen.clear()
        cache = pkg.GradientCache(torch.zeros(n, dtype=torch.float64, device="cuda"), x, "complex", max_batch=max_batch)
        df = torch.full((n,), NAN, dtype=torch.float64, device="cuda")
        pkg.finite_difference_gradient_(df, f, x, cache)
        torch.cuda.synchronize()
        assert len(seen) == len(ref["points"]) == ref["fcalls"] == n, what
        for k, (p, q) in enumerate(zip(seen, ref["points"])):
            assert_same_bits(p, q, f"{what}: point {k}")
        assert_same_bits(df, ref["df"], f"{what}: df")
        assert_same_bits(x, xh, f"{what}: x modified")


# ------------------------------------------------------------------------------------------------ gradient: graph replay
def _replay(pkg, g, x, df, cache, seq, code, fx_of):
    """run seq = [(EDGES index for x, relstep, dir, captured?)] through one graph-enabled cache; fx_of(xh, k) sets
    cache.fx (or the tensor it names) for call k and returns the number the restatement is given"""
    n = g.n
    for k, (first, relstep, dir, captured) in enumerate(seq):
        xh = edge_x(n, first, TILE_EDGES + (n - 1,))
        x.copy_(_cuda(xh))                                     # same storage, new values
        fxv = fx_of(xh, k)
        calls0 = g.ctx.calls
        pkg.finite_difference_gradient_(df, g.fn, x, cache, relstep=relstep, dir=dir)
        torch.cuda.synchronize()
        what = f"call {k}: x from EDGES[{first}], relstep={relstep}, dir={dir}, fx={fxv}"
        ref = so.gradient(g.twin.native("synth_guarded"), xh, code, fx=fxv, relstep=relstep, dir=dir)
        assert_same_bits(df, ref["df"], f"{what}: df")
        assert g.ctx.calls - calls0 == (ref["fcalls"] if captured else 0), \
            f"{what}: {'not ' if captured else ''}recaptured"
        assert cache._last_plan.counters()["jacobians"] == k + 1


@pytest.mark.parametrize("kind", ["number", "tensor"])
def test_gpu_gradient_graph_replay_follows_fx_and_x(pkg, kind):
    # a numeric cache.fx is staged in the cache's one device slot before every call: a replay must see the new number
    n = 33
    g = Guarded(pkg, n)
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    df = torch.full((n,), NAN, dtype=torch.float64, device="cuda")
    fx_t = torch.zeros(1, dtype=torch.float64, device="cuda")
    cache = pkg.GradientCache(fx_t if kind == "tensor" else 0.0, None, None, torch.zeros_like(x), "forward",
                              max_batch=64, use_graph=True)
    shifts = [0.0, 0.5, -3.0, 0.0, 0.25, 0.25]

    def fx_of(xh, k):
        v = float(f64(g.twin(xh)) + f64(shifts[k]))
        if kind == "tensor":
            fx_t.fill_(v)
        else:
            cache.fx = v
        return v

    seq = [(8, None, 1.0, True), (8, None, 1.0, False), (8, None, 1.0, False), (5, None, 1.0, False),
           (5, 1e-3, 1.0, True), (5, 1e-3, -1.0, True)]
    _replay(pkg, g, x, df, cache, seq, so.FORWARD, fx_of)
    if kind == "number":
        assert cache._fin.numel() == 1


@pytest.mark.parametrize("mode", ["forward", "central"])
def test_gpu_gradient_graph_replay_follows_x_and_signed_zero_steps(pkg, mode):
    # relstep = -0.0 (absstep defaults to it) steps a -0.0 component to -0.0, relstep = +0.0 to +0.0: in forward mode
    # df there is -Inf or NaN.  The two calls differ in the step's sign bit alone, and must not share a graph.
    n = 33
    g = Guarded(pkg, n)
    code = so.FORWARD if mode == "forward" else so.CENTRAL
    x = torch.empty(n, dtype=torch.float64, device="cuda")
    df = torch.full((n,), NAN, dtype=torch.float64, device="cuda")
    cache = pkg.GradientCache(torch.zeros_like(x), x, mode, max_batch=64, use_graph=True)
    xh = edge_x(n, 1, TILE_EDGES + (n - 1,))
    assert np.signbit(xh[0]) and xh[0] == 0
    if mode == "forward":
        d = [so.gradient(g.twin.native("synth_guarded"), xh, code, relstep=r)["df"] for r in (0.0, -0.0)]
        assert np.isinf(d[0][0]) and np.isnan(d[1][0])            # the sign of the zero step reaches df
    seq = [(1, 0.0, 1.0, True), (1, -0.0, 1.0, True), (1, 0.0, 1.0, True), (5, 0.0, 1.0, False), (1, None, 1.0, True),
           (0, None, 1.0, False)]
    if mode == "forward":                                      # dir = -1 flips every forward step: a new call
        seq += [(0, None, -1.0, True), (8, None, -1.0, False)]
    _replay(pkg, g, x, df, cache, seq, code, lambda xh, k: None)
