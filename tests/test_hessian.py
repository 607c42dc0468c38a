"""Dense Hessians of a scalar f (src/hessians.jl:202-292).

CPU: the C restatement (scalar_oracle/) against the reference's own Hessian tests (test/finitedifftests.jl:561-614) and,
bit for bit, against an independent line-by-line Python transcription on random problems with IEEE edge values.
GPU: fdb_hessian bit-compared with the restatement's own run (no step sizes fed in) over sizes, batch caps, value-buffer
chunks, strided H, reduced grids and graph replay; call counts, the points f sees, error paths and the closed form."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from _util import assert_same_bits, hessian_transcribed
from scalar_oracle import fd_scalar_oracle as so

f64 = np.float64


@pytest.fixture(scope="module")
def soracle():
    so.build()
    so.lib()
    return so


def err_func(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))))


# ------------------------------------------------------------------------------------------------ KATs (CPU)
def test_kat_sin_cos(soracle):
    # finitedifftests.jl:561-576
    x = np.random.default_rng(1).random(2)
    H_ref = np.array([[-np.sin(x[0]), 0.0], [0.0, -np.cos(x[1])]])
    r = soracle.hessian(lambda v: np.sin(v[0]) + np.cos(v[1]), x)
    assert err_func(r["H"], H_ref) < 1e-4
    assert r["fcalls"] == 2 * 2 * 2 + 1


def test_kat_half_sum_abs2_is_identity(soracle):
    # finitedifftests.jl:593-598
    r = soracle.hessian(lambda v: float(np.sum(np.abs(v) ** 2)) / 2, np.ones(2))
    np.testing.assert_allclose(r["H"], np.eye(2), atol=1e-8)


@pytest.mark.parametrize("cache_x", [None, np.arange(5.0, 9.0)])
def test_kat_issue_185_sum_abs2_exact(soracle, cache_x):
    # finitedifftests.jl:608-614: exactly Diagonal(2), also with a HessianCache built from another x
    x = np.arange(1.0, 5.0)
    f = soracle.SynthScalar(4)
    cache = None if cache_x is None else [cache_x.copy() for _ in range(4)]
    r = soracle.hessian(f.native("synth_sumsq"), x, cache=cache)
    assert np.array_equal(r["H"], np.diag(np.full(4, 2.0)))


def test_default_relstep_is_eps_quarter(soracle):
    assert soracle.default_relstep(3) == 2.0 ** -13 == np.finfo(float).eps ** 0.25


# ------------------------------------------------------------------------------------------------ transcription (CPU)
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-320, -1e-320, 5e-324, 1e300, -1e300, 1e-160, 1.0, -2.5]


def _poly(v):
    with np.errstate(all="ignore"):
        s = f64(0)
        for k in range(len(v)):
            s = s + f64(0.5) * v[k] * v[k] * v[k] + v[k] * v[(k + 1) % len(v)]
        return s


def test_oracle_matches_transcription_random(soracle):
    rng = np.random.default_rng(185)
    for trial in range(300):
        n = int(rng.integers(0, 6))
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)
        for k in range(n):
            if rng.random() < 0.3:
                x[k] = EDGES[rng.integers(len(EDGES))]
        relstep = [None, 0.0, 1e-3, float(10.0 ** rng.integers(-12, 0))][rng.integers(4)]
        absstep = [None, 0.0, 1e-6, 1e-320][rng.integers(4)]
        H, fx, pts = hessian_transcribed(_poly, x, relstep, absstep)
        r = soracle.hessian(_poly, x, relstep=relstep, absstep=absstep, log=True)
        assert r["fcalls"] == len(pts) == 2 * n * n + 1
        for p, q in zip(r["points"], pts):
            assert_same_bits(p, q, f"trial {trial}: point")
        assert_same_bits(r["H"][:n, :n], H, f"trial {trial}: H")
        assert_same_bits(np.array([r["fx"]]), np.array([fx]), f"trial {trial}: fx")


# ------------------------------------------------------------------------------------------------ GPU
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


class Quartic:
    """fdbs_quartic on the device and its CPU twin, a_i in [0.5, 1.5), w_i in [-1, 1), x from fdbs_fill_x."""

    def __init__(self, pkg, n, seed=7):
        rng = np.random.default_rng(seed + n)
        self.n = n
        self.a = 0.5 + rng.random(n)
        self.w = rng.random(n) * 2 - 1
        dev = torch.device("cuda:0")
        self.d_a = torch.from_numpy(self.a).to(dev)
        self.d_w = torch.from_numpy(self.w).to(dev)
        self.x = torch.empty(max(n, 1), dtype=torch.float64, device=dev)[:n]
        if n:
            pkg._lib.synth().fdbs_fill_x(self.x.data_ptr(), n, 0xC0FFEE + n, None)
        self.ctx = pkg._lib.ScalarCtx(n, self.d_a.data_ptr(), self.d_w.data_ptr(), 0)
        self.fn = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_quartic, C.c_void_p).value, self.ctx)
        self.twin = so.SynthScalar(n, self.a, self.w)

    def closed_form(self, x):
        n = self.n
        H = np.diag(12 * self.a * x * x) + np.outer(self.w, self.w) / n
        H[np.arange(n - 1), np.arange(1, n)] += 1
        H[np.arange(1, n), np.arange(n - 1)] += 1
        return H


_ORACLE = {}


def _oracle_run(q):
    if q.n not in _ORACLE:
        xh = q.x.cpu().numpy().copy()
        _ORACLE[q.n] = so.hessian(q.twin.native("synth_quartic"), xh)
    return _ORACLE[q.n]


def _device_H(pkg, q, *, ldH=None, use_graph=False, reps=1, **kw):
    n = q.n
    ld = n if ldH is None else ldH
    buf = torch.full((max(n, 1), max(ld, 1)), float("nan"), dtype=torch.float64, device="cuda")   # column j = buf[j]
    H = buf[:n, :n].t() if n else torch.empty((0, 0), dtype=torch.float64, device="cuda")
    cache = pkg.HessianCache(q.x, use_graph=use_graph, **kw)
    fx = torch.full((1,), float("nan"), dtype=torch.float64, device="cuda")
    x0 = q.x.clone()
    for _ in range(reps):
        pkg.finite_difference_hessian_(H, q.fn, q.x, cache, fx=fx)
    torch.cuda.synchronize()
    assert_same_bits(q.x, x0, "x modified", allow_nan=False)
    return H, buf, fx, cache._last_plan


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2, 3, 33, 257])
def test_gpu_hessian_bitexact_batches(pkg, n):
    q = Quartic(pkg, n)
    ref = _oracle_run(q)
    for mb in (1, 7, 64, 4096):
        q.ctx.calls = 0
        H, buf, fx, plan = _device_H(pkg, q, max_batch=mb)
        assert_same_bits(H.cpu().numpy(), ref["H"][:n, :n], f"n={n} max_batch={mb}", allow_nan=False)
        assert_same_bits(fx.cpu().numpy(), np.array([ref["fx"]]), "f(x)")
        c, info = plan.counters(), plan.info()
        assert q.ctx.calls == c["f_points"] == ref["fcalls"] == info["fcalls_per_jacobian"] == 2 * n * n + 1
        assert info["n_entries"] == n * n
        assert c["f_invocations"] >= -(-(2 * n * n + 1) // mb)


@pytest.mark.gpu
def test_gpu_hessian_bitexact_n1000(pkg):
    q = Quartic(pkg, 1000)
    H, _, _, plan = _device_H(pkg, q, max_batch=4096)
    assert_same_bits(H.cpu().numpy(), _oracle_run(q)["H"], "n=1000", allow_nan=False)
    assert plan.counters()["f_points"] == 2 * 1000 ** 2 + 1


@pytest.mark.gpu
@pytest.mark.parametrize("n,scratch", [(33, 8 * 300), (257, 8 * 5000), (257, 8)])
def test_gpu_hessian_value_chunks(pkg, n, scratch):
    q = Quartic(pkg, n)
    H, _, _, plan = _device_H(pkg, q, max_batch=64, scratch_bytes=scratch)
    assert plan.info()["n_groups"] > 1                     # several assembly chunks
    assert_same_bits(H.cpu().numpy(), _oracle_run(q)["H"], f"n={n} scratch={scratch}", allow_nan=False)


@pytest.mark.gpu
@pytest.mark.parametrize("n,ld", [(33, 40), (257, 300), (3, 4)])
def test_gpu_hessian_strided_H_padding_untouched(pkg, n, ld):
    q = Quartic(pkg, n)
    H, buf, _, _ = _device_H(pkg, q, ldH=ld, max_batch=64)
    assert_same_bits(H.cpu().numpy(), _oracle_run(q)["H"], f"n={n} ldH={ld}", allow_nan=False)
    assert torch.isnan(buf[:, n:]).all(), "padding rows beyond n were written"


@pytest.mark.gpu
@pytest.mark.parametrize("sm", ["1", "3"])
def test_gpu_hessian_reduced_grid(pkg, sm, monkeypatch, tmp_path):
    monkeypatch.setenv("FDB_SM_COUNT", sm)
    q = Quartic(pkg, 257)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        H, _, _, _ = _device_H(pkg, q, max_batch=64)
        # the last kernel record of a session can be missing from its trace when the session stops right after it, and
        # hess_assemble is the last launch: throwaway launches take that place
        pad = torch.empty(1, device="cuda")
        for _ in range(64):
            pad.fill_(0.0)
        torch.cuda.synchronize()
    assert_same_bits(H.cpu().numpy(), _oracle_run(q)["H"], f"FDB_SM_COUNT={sm}", allow_nan=False)
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    ev = [e for e in json.loads(trace.read_text())["traceEvents"] if "hess_assemble" in e.get("name", "")]
    assert ev, "no hess_assemble kernel in the trace"
    tiles = 9 * 10 // 2                                    # 257 rows: 9 tile rows, the lower triangle of tiles
    for e in ev:
        grid = e["args"]["grid"]
        assert grid[0] <= 8 * int(sm) < tiles, grid       # several tiles per block
    patches = [e for e in json.loads(trace.read_text())["traceEvents"] if "hess_patch" in e.get("name", "")]
    assert patches


@pytest.mark.gpu
def test_gpu_hessian_graph_replay(pkg):
    q = Quartic(pkg, 33)
    ref = _oracle_run(q)
    H, _, fx, plan = _device_H(pkg, q, max_batch=64, use_graph=True, reps=3)
    assert_same_bits(H.cpu().numpy(), ref["H"], "graph replay", allow_nan=False)
    assert_same_bits(fx.cpu().numpy(), np.array([ref["fx"]]), "f(x)")
    c = plan.counters()
    assert c["jacobians"] == 3 and c["f_points"] == 3 * (2 * 33 * 33 + 1)


@pytest.mark.gpu
def test_gpu_hessian_points_seen_by_f(pkg):
    n = 4
    q = Quartic(pkg, n)
    seen = []

    def f(x):
        seen.append(x.clone())
        return (x * x).sum()

    xh = q.x.cpu().numpy().copy()
    for mb in (1, 5):
        seen.clear()
        H = pkg.zeros_colmajor(n, n)
        pkg.finite_difference_hessian_(H, f, q.x, pkg.HessianCache(q.x, max_batch=mb))
        torch.cuda.synchronize()
        ref = so.hessian(lambda v: float(np.sum(v * v)), xh, log=True)
        assert len(seen) == len(ref["points"]) == 2 * n * n + 1
        for k, (a, b) in enumerate(zip(seen, ref["points"])):
            assert_same_bits(a.cpu().numpy(), b, f"point {k}", allow_nan=False)
        np.testing.assert_allclose(H.cpu().numpy(), 2 * np.eye(n), atol=1e-6)


@pytest.mark.gpu
def test_gpu_hessian_closed_form(pkg):
    q = Quartic(pkg, 257)
    H, _, _, _ = _device_H(pkg, q, max_batch=4096)
    Hc = q.closed_form(q.x.cpu().numpy())
    assert err_func(H.cpu().numpy(), Hc) / np.max(np.abs(Hc)) < 1e-4


@pytest.mark.gpu
def test_gpu_hessian_out_of_place_and_kat(pkg):
    # finitedifftests.jl:608-614 on the device: sum(abs2) at 1:4 is exactly Diagonal(2), with a cache from 5:8 too
    x = torch.arange(1.0, 5.0, dtype=torch.float64, device="cuda")
    ctx = pkg._lib.ScalarCtx(4, None, None, 0)
    f = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_sumsq, C.c_void_p).value, ctx)
    for cache in (None, pkg.HessianCache(torch.arange(5.0, 9.0, dtype=torch.float64, device="cuda"))):
        H = pkg.finite_difference_hessian(f, x, cache)
        assert torch.equal(H.cpu(), torch.diag(torch.full((4,), 2.0, dtype=torch.float64)))
        assert H.stride() == (1, 4)


@pytest.mark.gpu
def test_gpu_hessian_errors(pkg):
    L = pkg._lib
    x = torch.ones(3, dtype=torch.float64, device="cuda")
    H = pkg.zeros_colmajor(3, 3)
    for bad in ("central", "forward", "complex"):
        with pytest.raises(L.FdbError) as e:
            pkg.finite_difference_hessian_(H, lambda v: v.sum(), x, pkg.HessianCache(x, bad))
        assert e.value.status == L.FDB_ERR_UNSUPPORTED
    h = C.c_void_p()
    o = L.PlanOpts(fdtype=L.FDB_HCENTRAL)
    assert L.lib().fdb_hessian_plan_create(C.byref(h), 3, 2, C.byref(o)) == L.FDB_ERR_INVALID        # ldH < n
    with pytest.raises(L.FdbError) as e:
        pkg.finite_difference_hessian_(H, pkg.NativeFn(C.cast(L.synth().fdbs_fail, C.c_void_p).value), x)
    assert e.value.status == L.FDB_ERR_CALLBACK

    class Boom(Exception):
        pass

    def f(v):
        raise Boom()

    with pytest.raises(Boom):
        pkg.finite_difference_hessian_(H, f, x)
    with pytest.raises(TypeError):
        pkg.finite_difference_hessian_(H, lambda v: v.sum(), x.cpu())
    with pytest.raises(TypeError):
        pkg.HessianCache(x.cpu())
    # a Hessian plan is not a Jacobian plan and vice versa
    cache = pkg.HessianCache(x)
    plan = cache.plan_for(3, 3, x.device)
    assert L.lib().fdb_jacobian(plan.handle, C.cast(L.synth().fdbs_fail, C.c_void_p), None, x.data_ptr(), H.data_ptr(),
                                None, None, L.STEP_DEFAULT, L.STEP_DEFAULT, 1.0, None) == L.FDB_ERR_INVALID
    jh = C.c_void_p()
    assert L.lib().fdb_plan_create_dense(C.byref(jh), 3, 3, 3, C.byref(L.PlanOpts(fdtype=L.FDB_CENTRAL))) == L.FDB_OK
    jp = pkg.Plan(jh.value)
    assert L.lib().fdb_hessian(jp.handle, C.cast(L.synth().fdbs_fail, C.c_void_p), None, x.data_ptr(), H.data_ptr(), None,
                               L.STEP_DEFAULT, L.STEP_DEFAULT, None) == L.FDB_ERR_INVALID


@pytest.mark.gpu
def test_gpu_hessian_python_float_f(pkg):
    # f returning a plain Python float (a Julia-style f returns a native Float64): the value is stored as float64.
    # finitedifftests.jl:608-614: sum(abs2) at 1:4 is exactly Diagonal(2); the sum written out in Julia's order
    xh = np.arange(1.0, 5.0)
    x = torch.from_numpy(xh).cuda()
    f_host = lambda v: ((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]) + v[3] * v[3]
    ref = so.hessian(f_host, xh)
    assert np.array_equal(ref["H"], np.diag(np.full(4, 2.0)))

    def f_batched(X):
        return [float(f_host(X[b])) for b in range(X.shape[0])]
    f_batched.batched = True
    for f in (lambda v: float(f_host(v)), f_batched):
        H = pkg.finite_difference_hessian(f, x, pkg.HessianCache(x, max_batch=8))
        assert_same_bits(H.cpu().numpy(), ref["H"], "Python float f", allow_nan=False)
