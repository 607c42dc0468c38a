"""Host side of the block-banded plan (no GPU): which targets the mirror sends to fdb_plan_create_block_banded, and the
closed form the scatter kernel uses (slot -> block, row, colour), restated here and checked against the hook's entry
list (findstructralnz) and the block-cyclic colouring of matrix_colors."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


def _closed_form_slots(rb, l, u, lam, mu):
    """(rows, cols, slots) 1-based, walking the band data in storage order as diff_scatter_block_band does."""
    off = np.concatenate([[0], np.cumsum(rb)]).astype(np.int64)
    n, N = int(off[-1]), len(rb)
    sw, w = lam + mu + 1, (l + u + 1) * (lam + mu + 1)
    s = np.arange(w * n, dtype=np.int64)
    c, t = s // w, s % w
    b, d = t // sw, t % sw
    J = np.searchsorted(off, c, side="right") - 1          # the largest J with off[J] <= c
    j = c - off[J]
    K = J + b - u
    inK = (K >= 0) & (K < N)
    Kc = np.clip(K, 0, max(N - 1, 0))
    k = j + d - mu
    inside = inK & (k >= 0) & (k < off[Kc + 1] - off[Kc])
    rows = off[Kc] + k
    return rows[inside] + 1, c[inside] + 1, s[inside] + 1


@pytest.mark.parametrize("seed", range(40))
def test_closed_form_is_the_hook_entry_set(pkg, seed):
    rng = np.random.default_rng(seed)
    N = int(rng.integers(1, 13))
    rb = [int(v) for v in rng.integers(0 if seed % 5 == 0 else 1, 10, N)]     # some cases with empty blocks
    l, u, lam, mu = (int(v) for v in rng.integers(0, 5, 4))
    B = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device="cpu")
    rows, cols, slots = B.findstructralnz()
    r2, c2, s2 = _closed_form_slots(rb, l, u, lam, mu)
    o1, o2 = np.argsort(slots), np.argsort(s2)
    assert np.array_equal(slots[o1], s2[o2])
    assert np.array_equal(rows[o1], r2[o2]) and np.array_equal(cols[o1], c2[o2])


@pytest.mark.parametrize("seed", range(10))
def test_matrix_colors_is_the_block_cyclic_form(pkg, seed):
    rng = np.random.default_rng(100 + seed)
    rb = [int(v) for v in rng.integers(1, 8, int(rng.integers(1, 9)))]
    l, u, lam, mu = (int(v) for v in rng.integers(0, 4, 4))
    B = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device="cpu")
    off = np.concatenate([[0], np.cumsum(rb)])
    c = np.arange(B.n)
    J = np.searchsorted(off, c, side="right") - 1
    assert np.array_equal(B.matrix_colors() - 1, (J % (l + u + 1)) * (lam + mu + 1) + (c - off[J]) % (lam + mu + 1))


def test_routing(pkg, api):
    B = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 2), (0, 3), device="cpu")
    blocks, l, u, lam, mu, ldata = api._block_banded_plan_args(B, B)
    assert blocks.dtype == np.int64 and blocks.tolist() == [3, 4, 2]
    assert (l, u, lam, mu, ldata) == (1, 2, 0, 3, B.w * B.n)
    # the same structure in another object, and the mirror's BlockBandedMatrix
    S = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 2), (0, 3), device="cpu")
    assert api._block_banded_plan_args(B, S) is not None
    BB = pkg.BlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 1), device="cpu")
    assert api._block_banded_plan_args(BB, BB)[3:5] == (3, 3)
    # these keep the slot-addressed route
    assert api._block_banded_plan_args(torch.zeros(9, 9, dtype=torch.float64), B) is None       # dense J
    R = pkg.BandedBlockBandedMatrix([3, 4, 2], [2, 5, 2], (1, 1), (1, 1), device="cpu")
    assert api._block_banded_plan_args(R, R) is None                                           # rectangular blocks
    D = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 1), (1, 1), device="cpu")
    assert api._block_banded_plan_args(D, B) is None                                           # different structures
    Ng = pkg.BandedBlockBandedMatrix([3, 3], [3, 3], (-1, 1), (1, 1), data=torch.zeros(1), device="cpu")
    assert api._block_banded_plan_args(Ng, Ng) is None                                         # negative bandwidth
