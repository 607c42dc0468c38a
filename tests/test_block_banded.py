"""BandedBlockBandedMatrix targets (SURVEY.md §8f rank 3; ext/FiniteDiffBlockBandedMatricesExt.jl:16-42): the hook's
entry set through the generic slot-addressed path.  Shape of test/coloring_tests.jl:99-119 (2-D 5-point stencil, block
structure fill(g, g), bandwidths (1,1),(1,1)) at reduced grid size: Jbbb ≈ Jsparse, both from the same colouring."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sps
import torch

from _util import assert_same_bits, csc_to_dense


def f_lap5(g):
    def f(out, x):
        X = x.reshape(g, g, order="F")
        O = out.reshape(g, g, order="F")
        im = np.maximum(np.arange(g) - 1, 0)
        ip = np.minimum(np.arange(g) + 1, g - 1)
        O[:, :] = X + X[im, :] + X[ip, :] + X[:, im] + X[:, ip]
    return f


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


def _bbb(pkg, g, device="cpu"):
    return pkg.BandedBlockBandedMatrix([g] * g, [g] * g, (1, 1), (1, 1),
                                       data=torch.full((9 * g * g,), float("nan"), dtype=torch.float64, device=device))


def test_oracle_bbb_equals_csc_of_same_pattern(pkg, oracle):
    g = 12
    n = g * g
    B = _bbb(pkg, g)
    rows, cols, slots = B.findstructralnz()
    colors = B.matrix_colors()
    assert colors.max() == 9
    # the colouring is valid for the whole structure: no row holds two columns of one colour
    S = sps.csc_matrix((np.ones(len(rows)), (rows - 1, cols - 1)), shape=(n, n))
    Sr = S.tocsr()
    for r in range(n):
        cs = colors[Sr.indices[Sr.indptr[r]:Sr.indptr[r + 1]]]
        assert len(set(cs.tolist())) == len(cs)
    x = np.random.default_rng(1).random(n)
    data = np.full(9 * n, np.nan)
    r1 = oracle.jacobian(oracle.Problem.coo_to_slots(n, n, rows, cols, slots, 9 * n), data, f_lap5(g), x.copy(), colorvec=colors)
    assert r1["fcalls"] == 10
    S.sort_indices()
    colptr, rowval = S.indptr.astype(np.int64) + 1, S.indices.astype(np.int64) + 1
    nz = np.full(S.nnz, np.nan)
    oracle.jacobian(oracle.Problem.csc_same(n, n, colptr, rowval), nz, f_lap5(g), x.copy(), colorvec=colors)
    Jb = np.zeros((n, n))
    Jb[rows - 1, cols - 1] = data[slots - 1]
    assert_same_bits(Jb, csc_to_dense(n, n, colptr, rowval, nz), allow_nan=False)               # Jbbb == Jsparse (coloring_tests.jl:115)
    # and both equal the uncoloured dense Jacobian
    Jd = np.zeros(n * n)
    oracle.jacobian(oracle.Problem.dense(n, n), Jd, f_lap5(g), x.copy())
    np.testing.assert_allclose(Jb, Jd.reshape(n, n, order="F"), rtol=1e-6, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_gpu_bbb_bitexact(pkg, oracle, fdtype):
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    dev = torch.device("cuda:0")
    L = pkg._lib
    g = 40
    n = g * g
    B = _bbb(pkg, g, dev)
    rows, cols, slots = B.findstructralnz()
    colors = B.matrix_colors()
    x = torch.empty(n, dtype=torch.float64, device=dev)
    L.synth().fdbs_fill_x(x.data_ptr(), n, 77, None)
    ctx = L.Lap5Ctx(g, 0)
    f = pkg.NativeFn(C.cast(L.synth().fdbs_lap5, C.c_void_p).value, ctx)
    cache = pkg.JacobianCache(x, fdtype, colorvec=colors, sparsity=B)
    pkg.finite_difference_jacobian_(B, f, x, cache)
    torch.cuda.synchronize()
    ref = np.full(9 * n, np.nan)
    r = oracle.jacobian(oracle.Problem.coo_to_slots(n, n, rows, cols, slots, 9 * n), ref, oracle.native_fn("synth_lap5"),
                        oracle.fill_x(n, 77), fdtype=0 if fdtype == "forward" else 1, colorvec=colors,
                        eps_override=cache._last_plan.eps(), ctx=oracle.SynthLap5Ctx(g, 1))
    assert ctx.calls == r["fcalls"]
    got = B.data.cpu().numpy()
    # slots the structure does not address are zero (fill_matrix!), the others bit-identical
    touched = np.zeros(9 * n, bool)
    touched[slots - 1] = True
    assert_same_bits(got[touched], ref[touched], allow_nan=False)
    assert np.all(got[~touched] == 0)
    # cache-less entry picks the structured J as its own sparsity (jacobians.jl:455)
    B2 = _bbb(pkg, g, dev)
    pkg.finite_difference_jacobian_(B2, f, x, fdtype, colorvec=colors)
    assert_same_bits(B2.data.cpu().numpy()[touched], ref[touched], allow_nan=False)


def test_block_banded_dense_blocks_structure(pkg, oracle):
    # BlockBandedMatrix hook (ext/FiniteDiffBlockBandedMatricesExt.jl:44-68): every row of every in-band block
    g = 6
    n = g * g
    B = pkg.BlockBandedMatrix([g] * g, [g] * g, (1, 1), data=torch.zeros((3 * (2 * (g - 1) + 1)) * n, dtype=torch.float64))
    rows, cols, slots = B.findstructralnz()
    S = np.zeros((n, n), bool)
    S[rows - 1, cols - 1] = True
    bi = np.arange(n) // g
    assert np.array_equal(S, np.abs(np.subtract.outer(bi, bi)) <= 1)           # block tridiagonal, dense blocks
    assert len(np.unique(slots)) == len(slots) and slots.max() <= B.w * n
    colors = B.matrix_colors()
    x = np.random.default_rng(2).random(n)
    data = np.zeros(B.w * n)
    oracle.jacobian(oracle.Problem.coo_to_slots(n, n, rows, cols, slots, B.w * n), data, f_lap5(g), x.copy(), colorvec=colors)
    Jb = np.zeros((n, n))
    Jb[rows - 1, cols - 1] = data[slots - 1]
    Jd = np.zeros(n * n)
    oracle.jacobian(oracle.Problem.dense(n, n), Jd, f_lap5(g), x.copy())
    np.testing.assert_allclose(Jb, Jd.reshape(n, n, order="F"), rtol=1e-6, atol=1e-6)   # Jbb ≈ Jsparse (coloring_tests.jl:119)


def _literal_bbb_writes(rb, l, u, lam, mu, colorvec):
    """ext/FiniteDiffBlockBandedMatricesExt.jl:16-42 transcribed: for each colour, the (row, col, in-block slot) triples
    the hook stores to, in its own loop order (block column J, block row K in blockcolrange, column j, row k)."""
    N = len(rb)
    off = np.concatenate([[0], np.cumsum(rb)])
    out = {}
    for color_i in range(1, int(max(colorvec)) + 1):
        w = []
        for J in range(1, N + 1):
            c_v = colorvec[off[J - 1]:off[J]]                       # c.blocks[J]
            for K in range(max(1, J - u), min(N, J + l) + 1):       # blockcolrange(Jac, J)
                m, n = rb[K - 1], rb[J - 1]                         # size(view(Jac, K, J))
                for j in range(1, n + 1):
                    if c_v[j - 1] == color_i:
                        for k in range(max(1, j - mu), min(m, j + lam) + 1):
                            w.append((off[K - 1] + k, off[J - 1] + j, mu + k - j + 1))   # unsafe_store! offset in the column
        out[color_i] = w
    return out


def _literal_blockbanded_writes(rb, l, u, colorvec):
    """ext/FiniteDiffBlockBandedMatricesExt.jl:44-68 transcribed (dense blocks inside the block band)."""
    N = len(rb)
    off = np.concatenate([[0], np.cumsum(rb)])
    out = {}
    for color_i in range(1, int(max(colorvec)) + 1):
        w = []
        for J in range(1, N + 1):
            c_v = colorvec[off[J - 1]:off[J]]
            for j in range(1, rb[J - 1] + 1):
                if c_v[j - 1] == color_i:
                    for K in range(max(1, J - u), min(N, J + l) + 1):
                        for k in range(1, rb[K - 1] + 1):
                            w.append((off[K - 1] + k, off[J - 1] + j))
        out[color_i] = w
    return out


@pytest.mark.parametrize("seed", range(25))
def test_block_banded_entry_sets_match_literal_hooks_cpu(pkg, seed):
    # host logic only (no GPU): the entry sets the mirror hands to the slot-addressed scatter are exactly what the
    # reference's two block-banded hooks store to, colour by colour
    rng = np.random.default_rng(seed)
    N = int(rng.integers(1, 6))
    rb = [int(b) for b in rng.integers(1, 7, N)]
    l, u = int(rng.integers(0, 3)), int(rng.integers(0, 3))
    lam, mu = int(rng.integers(0, 4)), int(rng.integers(0, 4))
    n = sum(rb)
    cv = rng.integers(1, 5, n).astype(np.int64)
    B = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device="cpu")
    rows, cols, slots = B.findstructralnz()
    lit_w = _literal_bbb_writes(rb, l, u, lam, mu, cv)
    for color_i, w in lit_w.items():
        sel = cv[cols - 1] == color_i
        got = sorted(zip(rows[sel].tolist(), cols[sel].tolist()))
        assert got == sorted((r, c) for r, c, _ in w)
    assert len(set(slots.tolist())) == len(slots) and slots.min(initial=1) >= 1 and slots.max(initial=1) <= B.w * n
    # sub-band position inside the block's band column is the reference's unsafe_store! offset (mu + k - j + 1)
    sw = lam + mu + 1
    key = {(r, c): s for r, c, s in (t for w in lit_w.values() for t in w)}
    for r, c, s in zip(rows.tolist(), cols.tolist(), slots.tolist()):
        assert ((s - 1) % B.w) % sw + 1 == key[(r, c)]
    # dense blocks
    BB = pkg.BlockBandedMatrix(rb, rb, (l, u), device="cpu")
    r2, c2, s2 = BB.findstructralnz()
    lit2 = _literal_blockbanded_writes(rb, l, u, cv)
    for color_i, w in lit2.items():
        sel = cv[c2 - 1] == color_i
        assert sorted(zip(r2[sel].tolist(), c2[sel].tolist())) == sorted(w)
    assert len(set(s2.tolist())) == len(s2)
