"""The staged scatter's tile claiming across calls: every call of a plan covers every tile exactly once.

After its first tiles a block of diff_scatter_staged claims the next walk position from a counter the plan owns; the
launch's last claim re-arms it for the next launch, with no host step.  A counter left off zero would make the next
call skip tiles, so here one plan runs several calls in a row — eager, and replayed from its captured CUDA graph — with
J poisoned with NaN before each, at grids of 1 and 3 SMs' worth of blocks (tens of claimed tiles per block), in the band
and the indexed form, forward and central.  Every call must give J bit-identical to the oracle fed the device step sizes,
with no NaN left."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_same_bits, fdb_env, tridiag_csc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("no_band", [None, 1])
@pytest.mark.parametrize("sm_count", [1, 3])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_repeated_calls_cover_every_tile(pkg, fdtype, sm_count, no_band, use_graph):
    from oracle import fd_oracle as orc
    N = 40_001                                 # 120 001 entries: 117 full tiles and a partial one
    dev = torch.device("cuda:0")
    L = pkg._lib
    colptr, rowval = tridiag_csc(N)
    cv = (np.arange(N) % 3 + 1).astype(np.int64)
    x = torch.empty(N, dtype=torch.float64, device=dev)
    L.synth().fdbs_fill_x(x.data_ptr(), N, 0x5EED + 7, None)
    J = pkg.SparseMatrixCSC(N, N, torch.from_numpy(colptr), torch.from_numpy(rowval),
                            torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=dev))
    ctx = L.TridiagCtx(N, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_tridiag, C.c_void_p).value, ctx)
    with fdb_env(SM_COUNT=sm_count, NO_BAND=no_band):
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J, use_graph=use_graph)
        pkg.finite_difference_jacobian_(J, f, x, cache)
    torch.cuda.synchronize()
    info = cache._last_plan.info()
    assert info["staged"], info
    eps = cache._last_plan.eps()
    xh = orc.fill_x(N, 0x5EED + 7)
    ref = np.full(len(rowval), np.nan)
    orc.jacobian(orc.Problem.csc_same(N, N, colptr, rowval), ref, orc.native_fn("synth_tridiag"), xh,
                 fdtype=0 if fdtype == "forward" else 1, colorvec=cv, eps_override=eps,
                 ctx=orc.SynthTridiagCtx(N, 1))
    assert_same_bits(J.nzval, ref, f"{fdtype} call 1", allow_nan=False)
    for call in range(2, 5):
        J.nzval.fill_(float("nan"))
        pkg.finite_difference_jacobian_(J, f, x, cache)
        torch.cuda.synchronize()
        assert_same_bits(J.nzval, ref, f"{fdtype} call {call}", allow_nan=False)
