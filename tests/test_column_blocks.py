"""Column-block shards (SURVEY.md §8f row 4): a contiguous block of columns + the row / x ranges it touches, a
slice-aware f!, the step sizes of the FULL x supplied from outside.  Bar: every block's values are bit-identical to its
segment of the unsharded Jacobian (which test_gpu_parity.py pins bit-exactly on the oracle).  The blocks of one
problem are run one after the other on one GPU here; tests/test_gpu_multi.py runs them one per process."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from _util import assert_same_bits, cyc_colors, tridiag_csc  # noqa: E402


def test_column_blocks_balance_entries_cpu():
    import _bootstrap
    _bootstrap.load_package()
    from finitediff_jl_b200 import distributed as fdist
    colptr, _ = tridiag_csc(1000)
    b = fdist.column_blocks(colptr, 4)
    assert b[0] == 0 and b[-1] == 1000 and all(b[i] <= b[i + 1] for i in range(4))
    per = [int(colptr[b[i + 1]] - colptr[b[i]]) for i in range(4)]
    assert max(per) - min(per) <= 3                       # a column holds at most 3 entries
    assert fdist.column_blocks(colptr, 1) == [0, 1000]
    # more ranks than columns: trailing blocks are empty, boundaries stay monotone
    cp2, _ = tridiag_csc(2)
    b2 = fdist.column_blocks(cp2, 4)
    assert b2[0] == 0 and b2[-1] == 2 and all(b2[i] <= b2[i + 1] for i in range(4))


@pytest.mark.parametrize("seed,world", [(0, 1), (1, 2), (2, 3), (3, 5), (4, 8)])
def test_block_geometry_cpu(seed, world):
    # pure host logic of the column-block shards on CPU tensors: the blocks tile nzval, every block's rows / x hull
    # contain everything its slice-aware f! needs, the local pattern is the block's pattern rebased
    import scipy.sparse as sps
    import _bootstrap
    _bootstrap.load_package()
    from finitediff_jl_b200 import distributed as fdist
    rng = np.random.default_rng(seed)
    m, n = 61, 53
    bw_lo, bw_hi = int(rng.integers(0, 6)), int(rng.integers(0, 6))
    D = np.zeros((m, n), bool)
    for c in range(n):
        for r in range(max(0, c - bw_hi), min(m, c + bw_lo + 1)):
            D[r, c] = rng.random() < 0.7
    D[:, rng.integers(0, n)] = False                                   # an empty column
    A = sps.csc_matrix(D)
    A.sort_indices()
    colptr = torch.from_numpy(A.indptr.astype(np.int64) + 1)
    rowval = torch.from_numpy(A.indices.astype(np.int64) + 1)
    bounds = fdist.column_blocks(colptr, world)
    covered = np.zeros(A.nnz, int)
    for r in range(world):
        c0, c1 = bounds[r], bounds[r + 1]
        g = fdist.block_geometry(colptr, rowval, c0, c1)
        covered[g["p0"]:g["p1"]] += 1
        assert g["x0"] <= c0 and c1 <= g["x1"]
        sub = D[:, c0:c1]
        if sub.any():
            rows = np.nonzero(sub.any(axis=1))[0]
            assert g["r0"] == rows.min() and g["r1"] == rows.max() + 1
            need = np.nonzero(D[g["r0"]:g["r1"], :].any(axis=0))[0]    # columns the rows [r0, r1) depend on
            assert g["x0"] <= need.min() and need.max() < g["x1"]
        else:
            assert g["p0"] == g["p1"] and g["r0"] == g["r1"]
        # local pattern == the block's columns of D, rows rebased, placed at columns [c0 - x0, c1 - x0) of the slice
        cpl, rvl = g["colptr_loc"].numpy(), g["rowval_loc"].numpy()
        assert len(cpl) == g["x1"] - g["x0"] + 1 and cpl[0] == 1 and cpl[-1] == g["p1"] - g["p0"] + 1
        loc = np.zeros((max(g["r1"] - g["r0"], 0), g["x1"] - g["x0"]), bool)
        for jl in range(g["x1"] - g["x0"]):
            for q in range(cpl[jl] - 1, cpl[jl + 1] - 1):
                loc[rvl[q] - 1, jl] = True
        expect = np.zeros_like(loc)
        expect[:, c0 - g["x0"]:c1 - g["x0"]] = D[g["r0"]:g["r1"], c0:c1]
        assert np.array_equal(loc, expect)
    assert (covered == 1).all()


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


def _native(pkg, name, ctx):
    return pkg.NativeFn(C.cast(getattr(pkg._lib.synth(), name), C.c_void_p).value, ctx, max_batch=1)


@pytest.mark.gpu
@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("n,world", [(10007, 3), (64, 4), (5, 4)])
def test_tridiagonal_blocks_bit_identical(pkg, fdtype, n, world):
    from finitediff_jl_b200 import distributed as fdist
    dev = torch.device("cuda:0")
    colptr, rowval = tridiag_csc(n)
    cv = cyc_colors(n, 3)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 21, None)
    cp, rv = torch.from_numpy(colptr).to(dev), torch.from_numpy(rowval).to(dev)
    nnz = len(rowval)
    # unsharded
    J = pkg.SparseMatrixCSC(n, n, cp, rv, torch.full((nnz,), float("nan"), dtype=torch.float64, device=dev))
    ctx = pkg._lib.TridiagCtx(n, 0)
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=J)
    pkg.finite_difference_jacobian_(J, _native(pkg, "fdbs_tridiag", ctx), x, cache)
    eps_full = cache._last_plan.eps()
    # blocks, one after the other
    Jb = pkg.SparseMatrixCSC(n, n, cp, rv, torch.full((nnz,), float("nan"), dtype=torch.float64, device=dev))
    ep = fdist.EpsPlan(n, cv, fdtype, dev)
    eps = ep.compute(x)
    assert_same_bits(eps.cpu().numpy()[:3], eps_full, allow_nan=False)
    bounds = fdist.column_blocks(colptr, world)
    ctxs = []

    def factory(r0, r1, x0, x1):
        c = pkg._lib.TridiagRowsCtx(n, r0, r1 - r0, x0, 0)
        ctxs.append(c)
        return _native(pkg, "fdbs_tridiag_rows", c)

    calls = 0
    for r in range(world):
        blk = fdist.ColumnBlockJacobian(Jb, cv, fdtype, bounds[r], bounds[r + 1], dev, factory)
        assert blk.x0 <= blk.c0 and blk.c1 <= blk.x1 and blk.x1 - blk.x0 <= (blk.c1 - blk.c0) + 4
        blk.run(x, eps)
        torch.cuda.synchronize()
        if blk.c1 > blk.c0:
            c_loc = int(max(cv[blk.x0:blk.x1]))             # the colour loop runs 1:maximum(colorvec) of the slice
            assert ctxs[-1].calls == (1 + c_loc if fdtype == "forward" else 2 * c_loc)
        calls += ctxs[-1].calls
    assert_same_bits(Jb.nzval, J.nzval, allow_nan=False)                   # bit-identical, every slot written exactly once
    assert not torch.isnan(Jb.nzval).any()


@pytest.mark.gpu
def test_pentadiagonal_python_callable_blocks(pkg):
    # a Python slice-aware f!: rows [r0, r1) of a 5-band stencil from x[x0:x1]; colours j mod 5
    import scipy.sparse as sps
    from finitediff_jl_b200 import distributed as fdist
    dev = torch.device("cuda:0")
    n = 301
    A = sps.diags([np.ones(n - abs(k)) for k in (-2, -1, 0, 1, 2)], [-2, -1, 0, 1, 2], format="csc")
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    cv = cyc_colors(n, 5)
    w = torch.tensor([0.5, -1.0, 3.0, 2.0, -0.25], dtype=torch.float64, device=dev)
    x = torch.rand(n, dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(3)) + 0.5

    def rows(fx, xs, r0, r1, x0):
        # fx[i] = sum_k w[k] * x[r + k - 2]^2 over the in-range neighbours of global row r = r0 + i
        r = torch.arange(r0, r1, device=dev)
        acc = torch.zeros(r1 - r0, dtype=torch.float64, device=dev)
        for k in range(5):
            j = r + k - 2
            ok = (j >= 0) & (j < n)
            acc = acc + torch.where(ok, w[k] * xs[(j - x0).clamp(0, xs.numel() - 1)] ** 2, torch.zeros_like(acc))
        fx.copy_(acc)

    cp, rv = torch.from_numpy(colptr).to(dev), torch.from_numpy(rowval).to(dev)
    J = pkg.SparseMatrixCSC(n, n, cp, rv, torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=J)
    pkg.finite_difference_jacobian_(J, lambda fx, xx: rows(fx, xx, 0, n, 0), x, cache)
    Jb = pkg.SparseMatrixCSC(n, n, cp, rv, torch.full((A.nnz,), float("nan"), dtype=torch.float64, device=dev))
    eps = fdist.EpsPlan(n, cv, "forward", dev).compute(x)
    bounds = fdist.column_blocks(colptr, 3)
    for r in range(3):
        blk = fdist.ColumnBlockJacobian(Jb, cv, "forward", bounds[r], bounds[r + 1], dev,
                                        lambda r0, r1, x0, x1: (lambda fx, xs: rows(fx, xs, r0, r1, x0)))
        blk.run(x, eps)
    torch.cuda.synchronize()
    assert_same_bits(Jb.nzval, J.nzval, allow_nan=False)
    # and the values are the analytic derivative 2 w[k] x_j to forward-difference accuracy
    dense = torch.zeros(n, n, dtype=torch.float64)
    col_of = np.repeat(np.arange(n), np.diff(colptr))
    dense[torch.from_numpy(rowval - 1), torch.from_numpy(col_of)] = Jb.nzval.cpu()
    xc = x.cpu()
    for k in range(5):
        for r_ in (0, 1, 150, 299, 300):
            j = r_ + k - 2
            if 0 <= j < n:
                assert abs(float(dense[r_, j]) - 2 * float(w[k]) * float(xc[j])) < 1e-6
