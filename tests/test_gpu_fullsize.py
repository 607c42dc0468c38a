"""Parity AT the BASELINE.json sizes and on the branches only large shapes reach (run with -m gpu on an H100).

    C3  N = 10^6 5-point stencil, BandedMatrix l = u = 1000 (16 GB of band data): ~260 sampled columns (edges included)
        bit-compared with the oracle restricted to those columns' in-band slots, corner slots checked for zeros
    C4  N = 5*10^6 random sparse, 64 colours, nnz = 4*10^7: the WHOLE nzval bit-compared with the oracle — fused pass and
        colour-major lists
    C5  m = n = 10^5 dense, central, batch 256: a 511-column block (world = 196, rank 0) bit-compared with the oracle's
        dense branch over the same columns
    band with l+u+1 > 2049 (the flat band kernel's CH = 2048 < w-1 chunking), dense with m > 2048 (several row blocks
    per column in diff_columns) and batch 256, the windowed eps pass with C > 512 on a random pattern, dense J view with
    ldJ > m (padding rows untouched), sparsity=None with a non-default colorvec (the reference's quirk as written).

The oracle is fed the device-computed step sizes (bit-level eps is unpinned: Julia's norm is OpenBLAS dnrm2).
"""
import ctypes as C
import os
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from _util import assert_same_bits, cyc_colors  # noqa: E402

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


def native(pkg, name, ctx, max_batch=1):
    return pkg.NativeFn(C.cast(getattr(pkg._lib.synth(), name), C.c_void_p).value, ctx, max_batch=max_batch)


def host_threads():
    import bench
    return bench.usable_cores()


def free_gb():
    free, _ = torch.cuda.mem_get_info()
    return free / 2**30


def lap5_colors_np(g):
    idx = np.arange(g * g, dtype=np.int64)
    return ((idx % g) + 2 * (idx // g)) % 5 + 1


# ---------------------------------------------------------------------------------------------------- C3 full size
@pytest.mark.parametrize("fdtype", ["forward"])
def test_c3_full_size_sampled_columns_bitexact(pkg, oracle, dev, fdtype):
    if free_gb() < 40:
        pytest.skip("needs ~20 GB of free device memory")
    g = 1000
    n, l, u = g * g, g, g
    w = l + u + 1
    cv = lap5_colors_np(g)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0x5EED + 3, None)
    J = pkg.BandedMatrix(n, n, l, u, device=dev)
    J.data.fill_(float("nan"))
    ctx = pkg._lib.Lap5Ctx(g, 0)
    cache = pkg.JacobianCache(x, fdtype, colorvec=torch.from_numpy(cv).to(dev), sparsity=J)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_lap5", ctx), x, cache)
    torch.cuda.synchronize()
    eps = cache._last_plan.eps()
    assert ctx.calls == (6 if fdtype == "forward" else 10)
    # sampled columns: both ends (clipped bands, corner slots), around multiples of g, and random interior ones
    rng = np.random.default_rng(7)
    cols = np.unique(np.concatenate([np.arange(0, 8), np.arange(g - 3, g + 4), np.arange(n - 8, n),
                                     np.arange(n - g - 3, n - g + 4), rng.integers(0, n, 220)]))
    # oracle restricted to those columns: a CSC sparsity holding exactly their in-band rows (same colour loop, same
    # quotient vectors; `J[r,c] = vfx1[r]` for every listed (r,c) of the colour — what the banded hook stores there)
    counts = np.zeros(n, np.int64)
    r_lo = np.maximum(cols - u, 0)
    r_hi = np.minimum(cols + l, n - 1)
    counts[cols] = r_hi - r_lo + 1
    colptr = np.concatenate([[1], 1 + np.cumsum(counts)]).astype(np.int64)
    rowval = np.concatenate([np.arange(a, b + 1) for a, b in zip(r_lo, r_hi)]).astype(np.int64) + 1
    ref = np.full(len(rowval), np.nan)
    xh = oracle.fill_x(n, 0x5EED + 3)
    assert_same_bits(xh, x.cpu().numpy(), allow_nan=False)
    oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_lap5"), xh, fdtype=FD[fdtype],
                    colorvec=cv, eps_override=eps, ctx=oracle.SynthLap5Ctx(g, 1), nthreads=host_threads())
    p = 0
    for c, a, b in zip(cols, r_lo, r_hi):
        col = J.data[c * w:(c + 1) * w].cpu().numpy()
        k = b - a + 1
        d0 = u + a - c                                    # slot of row a:  u + r - c
        assert_same_bits(col[d0:d0 + k], ref[p:p + k], f"column {c}", allow_nan=False)
        assert not col[:d0].any() and not col[d0 + k:].any(), f"corner slots of column {c} must be 0"
        p += k
    # nothing left undefined anywhere in the 16 GB
    bad = 0
    step = 1 << 27
    for i in range(0, J.data.numel(), step):
        bad += int(torch.isnan(J.data[i:i + step]).sum())
    assert bad == 0


# ---------------------------------------------------------------------------------------------------- C4 full size
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_c4_full_size_bitexact(pkg, oracle, dev, strategy):
    """strategy 0 = auto (random pattern, one GPU: colour-major lists with every slab resident when one slab + f(x) fit
    the L2, else the storage-order pass), 1 = storage-order pass, 2 = colour-major lists per group, 3 = colour-major lists,
    one launch"""
    import bench
    fdtype = "forward"
    prob = bench.build_gpu_problem(pkg, "c4", fdtype, dev, 0, 1, 1, use_graph=False, strategy=strategy)
    J, f, x, cache = prob["J"], prob["f"], prob["x"], prob["cache"]
    pkg.finite_difference_jacobian_(J, f, x, cache)
    torch.cuda.synchronize()
    plan = cache._last_plan
    info = plan.info()
    lists_fit_l2 = 16 * prob["n"] <= torch.cuda.get_device_properties(dev).L2_cache_size
    lists = strategy in (2, 3) or (strategy == 0 and lists_fit_l2)
    assert info["strategy"] == (1 if lists else 0)
    assert info["lists_resident"] == (1 if strategy == 3 or (strategy == 0 and lists) else 0)
    assert info["n_groups"] == (64 if strategy == 2 else 1)
    eps = plan.eps()
    n, K = prob["n"], 8
    d_cols, d_coef, cv_t = prob["keep"]
    colsT, coefT = d_cols.cpu().numpy(), d_coef.cpu().numpy()
    colptr, rowval = J.colptr.cpu().numpy(), J.rowval.cpu().numpy()
    cv = cv_t.cpu().numpy()
    nt = host_threads()
    octx = oracle.SynthEllCtx(n, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), nt)
    ref = np.full(n * K, np.nan)
    xh = oracle.fill_x(n, 0x5EED + 4, nt)
    assert_same_bits(xh, x.cpu().numpy(), allow_nan=False)
    r = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_ellrows"), xh,
                        fdtype=FD[fdtype], colorvec=cv, eps_override=eps, ctx=octx, nthreads=nt)
    assert r["fcalls"] == 65 and prob["ctx"].calls == 65
    got = J.nzval.cpu().numpy()
    assert_same_bits(got, ref, allow_nan=False)
    assert np.isfinite(got).all() and np.count_nonzero(got) > 0.99 * got.size


# ---------------------------------------------------------------------------------------------------- C5 column block
def test_c5_column_block_bitexact(pkg, oracle, dev):
    """m = n = 10^5, central, batch 256 (the bench's batch): rank 0 of 196 owns columns [0, 511)."""
    L = pkg._lib
    n, mb, world = 100_000, 256, 196
    w = torch.rand(n, dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    bs = torch.zeros(((n + 1023) // 1024) * mb, dtype=torch.float64, device=dev)
    ctx = L.Rank1Ctx(n, w.data_ptr(), bs.data_ptr(), mb, 0)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    L.synth().fdbs_fill_x(x.data_ptr(), n, 0x5EED + 5, None)
    o = L.PlanOpts(fdtype=1, device=0, max_batch=mb, rank=0, world=world)
    h = C.c_void_p()
    L.check(L.lib().fdb_plan_create_dense(C.byref(h), n, n, n, C.byref(o)))
    plan = pkg.Plan(h.value)
    b, e = plan.dense_range()
    assert (b, e) == (0, 511)
    Jslab = torch.full((n * (e - b),), float("nan"), dtype=torch.float64, device=dev)
    L.check(L.lib().fdb_jacobian(plan.handle, C.cast(L.synth().fdbs_rank1, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p),
                                 x.data_ptr(), Jslab.data_ptr(), None, None, float("nan"), float("nan"), 1.0, None))
    torch.cuda.synchronize()
    assert ctx.calls == 2 * (e - b)
    # the oracle's dense branch over the leading 511 components: sparsity=nothing with maximum(colorvec) = 511
    # (jacobians.jl:589-598 loops color_i in 1:maximum(colorvec) and perturbs component color_i)
    cv = np.minimum(np.arange(1, n + 1, dtype=np.int64), e - b)
    wh = w.cpu().numpy()
    ref = np.full(n * (e - b), np.nan)
    r = oracle.jacobian(oracle.Problem.dense(n, n), ref, oracle.native_fn("synth_rank1"), oracle.fill_x(n, 0x5EED + 5), fdtype=1,
                        colorvec=cv, ctx=oracle.SynthRank1Ctx(n, wh.ctypes.data_as(C.POINTER(C.c_double)), 1))
    assert r["fcalls"] == 2 * (e - b)
    assert_same_bits(plan.eps(), r["eps"], allow_nan=False)
    assert_same_bits(Jslab.cpu().numpy(), ref, allow_nan=False)


# ---------------------------------------------------------------------------------------------------- large-shape branches
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_band_wider_than_2049_bitexact(pkg, oracle, dev, fdtype):
    """l+u+1 = 2201 > 2049: the flat band kernel cuts columns into several 2048-slot chunks (CH < w-1); every earlier
    test had one chunk per column."""
    g = 70
    n, l, u = g * g, 1100, 1100
    cv = lap5_colors_np(g)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 11, None)
    J = pkg.BandedMatrix(n, n, l, u, device=dev)
    J.data.fill_(float("nan"))
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_lap5", pkg._lib.Lap5Ctx(g, 0)), x, cache)
    torch.cuda.synchronize()
    ref = np.full((l + u + 1) * n, np.nan)
    oracle.jacobian(oracle.Problem.banded(n, n, l, u), ref, oracle.native_fn("synth_lap5"), oracle.fill_x(n, 11), fdtype=FD[fdtype],
                    colorvec=cv, eps_override=cache._last_plan.eps(), ctx=oracle.SynthLap5Ctx(g, 1))
    assert_same_bits(J.data.cpu().numpy(), ref, allow_nan=False)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_dense_many_row_blocks_batch_256_bitexact(pkg, oracle, dev, fdtype):
    """m = 6000 > 2048 rows (gridDim.x > 1 in diff_columns), batch 256 (the C5 bench batch)."""
    n, batch = 6000, 256
    w = np.random.default_rng(3).random(n)
    d_w = torch.from_numpy(w).to(dev)
    bs = torch.zeros(((n + 1023) // 1024) * batch, dtype=torch.float64, device=dev)
    ctx = pkg._lib.Rank1Ctx(n, d_w.data_ptr(), bs.data_ptr(), batch, 0)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 13, None)
    J = pkg.zeros_colmajor(n, n, dev)
    J.fill_(float("nan"))
    cache = pkg.JacobianCache(x, fdtype, max_batch=batch)
    pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_rank1", ctx, batch), x, cache)
    torch.cuda.synchronize()
    ref = np.zeros(n * n)
    r = oracle.jacobian(oracle.Problem.dense(n, n), ref, oracle.native_fn("synth_rank1"), oracle.fill_x(n, 13), fdtype=FD[fdtype],
                        ctx=oracle.SynthRank1Ctx(n, w.ctypes.data_as(C.POINTER(C.c_double)), 1), nthreads=host_threads())
    assert ctx.calls == r["fcalls"]
    assert_same_bits(J.cpu().numpy().reshape(-1, order="F"), ref, allow_nan=False)


def test_windowed_eps_random_pattern_700_colors(pkg, oracle, dev):
    """C = 700 > 512 (two windows of the shared-memory eps pass, uint16 colours) on a RANDOM pattern"""
    import scipy.sparse as sps
    Cc, K = 700, 6
    n = Cc * 40
    rng = np.random.default_rng(5)
    colors = np.argsort(rng.random((n, Cc)), axis=1)[:, :K]
    cols = (rng.integers(0, n // Cc, size=(n, K)) * Cc + colors).astype(np.int32)
    coef = rng.uniform(-1, 1, size=(n, K))
    A = sps.csc_matrix((np.ones(n * K), (np.repeat(np.arange(n), K), cols.reshape(-1))), shape=(n, n))
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    cv = cyc_colors(n, Cc)
    colsT, coefT = np.ascontiguousarray(cols.T), np.ascontiguousarray(coef.T)
    d_cols, d_coef = torch.from_numpy(colsT).to(dev), torch.from_numpy(coefT).to(dev)
    octx = oracle.SynthEllCtx(n, K, colsT.ctypes.data_as(C.POINTER(C.c_int32)), coefT.ctypes.data_as(C.POINTER(C.c_double)), 1)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 17, None)
    xh = oracle.fill_x(n, 17)
    for strategy in (1, 2):
        ctx = pkg._lib.EllCtx(n, K, d_cols.data_ptr(), d_coef.data_ptr(), 0)
        J = pkg.SparseMatrixCSC(n, n, torch.from_numpy(colptr), torch.from_numpy(rowval),
                                torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
        cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J, strategy=strategy)
        pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_ellrows", ctx), x, cache)
        torch.cuda.synchronize()
        eps = cache._last_plan.eps()
        assert cache._last_plan.info()["color_bits"] == 16
        ref = np.full(A.nnz, np.nan)
        own = oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), np.zeros(A.nnz), oracle.native_fn("synth_ellrows"),
                              xh.copy(), colorvec=cv, ctx=octx)
        np.testing.assert_allclose(eps, own["eps"], rtol=1e-14)
        oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), ref, oracle.native_fn("synth_ellrows"), xh.copy(),
                        colorvec=cv, eps_override=eps, ctx=octx)
        assert_same_bits(J.nzval.cpu().numpy(), ref, allow_nan=False)


# ---------------------------------------------------------------------------------------------------- ADVICE r1 / VERDICT r1 items
def test_dense_view_with_padding_rows(pkg, oracle, dev):
    """J is a strided column-major view (ldJ > m): fill_matrix!(J, 0) and the host copy touch rows [0, m) only."""
    from _util import tridiag_csc
    N, ld = 41, 48
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    store = torch.full((N, ld), 7.25, dtype=torch.float64, device=dev)       # column c at store[c, :], rows 0..ld
    Jview = store.t()[:N, :]                                                 # logical (N, N), strides (1, ld)
    assert Jview.stride() == (1, ld)
    x = torch.empty(N, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), N, 3, None)
    sp = pkg.SparseMatrixCSC(N, N, torch.from_numpy(colptr), torch.from_numpy(rowval), None)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=sp)
    pkg.finite_difference_jacobian_(Jview, native(pkg, "fdbs_tridiag", pkg._lib.TridiagCtx(N, 0)), x, cache)
    torch.cuda.synchronize()
    ref = np.zeros(N * N)
    oracle.jacobian(oracle.Problem.csc_to_dense(N, N, colptr, rowval), ref, oracle.native_fn("synth_tridiag"), oracle.fill_x(N, 3),
                    colorvec=cv, eps_override=cache._last_plan.eps(), ctx=oracle.SynthTridiagCtx(N, 1))
    got = store.cpu().numpy()
    assert_same_bits(got[:, :N].T.reshape(-1, order="F"), ref, allow_nan=False)
    assert (got[:, N:] == 7.25).all(), "padding rows between the columns do not belong to J"
    # host-buffer entry point with the same strided layout
    L = pkg._lib
    plan = cache._last_plan
    xh = pkg.pinned_empty(N)
    xh[:] = oracle.fill_x(N, 3)
    Jh = pkg.pinned_empty(N * ld)
    Jh[:] = 7.25
    ctx = L.TridiagCtx(N, 0)
    L.check(L.lib().fdb_jacobian_host(plan.handle, C.cast(L.synth().fdbs_tridiag, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p),
                                      xh.ctypes.data, Jh.ctypes.data, None, None, float("nan"), float("nan"), 1.0))
    hv = np.array(Jh).reshape(N, ld)
    assert_same_bits(hv[:, :N].T.reshape(-1, order="F"), ref, allow_nan=False)
    assert (hv[:, N:] == 7.25).all()


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_sparsity_nothing_with_colorvec_quirk(pkg, oracle, dev, fdtype):
    """sparsity=None + a non-default colorvec, as jacobians.jl:547-557 / :589-598 are written: component color_i is
    perturbed for color_i in 1:maximum(colorvec); J[:, 1:max] written, later columns untouched (no fill_matrix!)."""
    n = 12
    cv = np.array([1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2, 3], dtype=np.int64)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 23, None)
    xh = oracle.fill_x(n, 23)
    J = pkg.zeros_colmajor(n, n, dev)
    J.fill_(-3.5)
    calls = [0]

    def f(fx, xx):
        calls[0] += 1
        fx.copy_(torch.sin(xx) + xx.sum() * 0.25)

    cache = pkg.JacobianCache(x, fdtype, colorvec=cv)
    pkg.finite_difference_jacobian_(J, f, x, cache)
    torch.cuda.synchronize()
    got = J.cpu().numpy()
    assert calls[0] == (4 if fdtype == "forward" else 6)
    assert (got[:, 3:] == -3.5).all()
    ref = np.full(n * n, -3.5)

    def fh(fx, xx):
        fx[:] = np.sin(xx) + xx.sum() * 0.25

    r = oracle.jacobian(oracle.Problem.dense(n, n), ref, fh, xh.copy(), fdtype=FD[fdtype], colorvec=cv)
    assert r["fcalls"] == calls[0]
    refm = ref.reshape(n, n, order="F")
    assert (refm[:, 3:] == -3.5).all()
    np.testing.assert_allclose(got[:, :3], refm[:, :3], rtol=0, atol=1e-7)   # torch vs numpy sin/sum differ in the last bits
    with pytest.raises(pkg._lib.FdbError):                                  # maximum(colorvec) > n: BoundsError upstream
        pkg.finite_difference_jacobian_(pkg.zeros_colmajor(n, n, dev), f, x, pkg.JacobianCache(x, fdtype, colorvec=cv + n))


def test_explicit_zero_steps_pass_through(pkg, oracle, dev):
    """absstep = 0 is a pure relative step, relstep = 0 a pure absolute one (epsilons.jl:26-29); only 'keyword not given'
    selects the defaults."""
    from _util import tridiag_csc
    N = 300
    colptr, rowval = tridiag_csc(N)
    cv = cyc_colors(N, 3)
    x = torch.empty(N, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), N, 29, None)
    xh = oracle.fill_x(N, 29)
    for kw in (dict(relstep=1e-7, absstep=0.0), dict(relstep=0.0, absstep=1e-6)):
        J = pkg.SparseMatrixCSC(N, N, torch.from_numpy(colptr), torch.from_numpy(rowval),
                                torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
        cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J)
        pkg.finite_difference_jacobian_(J, native(pkg, "fdbs_tridiag", pkg._lib.TridiagCtx(N, 0)), x, cache, **kw)
        torch.cuda.synchronize()
        eps = cache._last_plan.eps()
        norms = np.array([np.sqrt(np.sqrt((xh[k::3] ** 2).sum())) for k in range(3)])
        want = np.maximum(kw["relstep"] * norms, kw["absstep"])
        np.testing.assert_allclose(eps, want, rtol=1e-13)
